"""Cost of ``--cam_trans epnp`` (RANSAC around EPnP on the GPU, csrc/pnp.cu) against the default closed form and against
the host loop of ``--cam_trans pnp``, on cfg2-like batches: 64 synthetic 512x512 frames, about 350 people planted with
``center_override``, bf16, synthetic weights.

    python tools/cam_trans_profile.py [--batch 64] [--iters 7]

Reports (median of --iters runs after one warm-up run):
  forward_batch_ms_lsq / forward_batch_ms_epnp : host wall clock of ROMP.forward_batch with each estimator;
  cam_trans_pnp_us_per_batch : device time of cam_trans_pnp_kernel per batch, from torch.profiler in a separate run;
  host_pnp_ms_per_batch : estimate_translation_pnp (cv2.solvePnPRansac per person, --cam_trans pnp) on the same joints.
The card name and power limit (read-only queries) are printed beside the numbers.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from romp_b200 import ROMP, romp_settings, synth  # noqa: E402
from romp_b200.main import estimate_translation_pnp  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [x.strip() for x in q.split(",")]
    except Exception:
        name, power = torch.cuda.get_device_name(0), "unknown"
    return name, power


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--iters", type=int, default=7)
    a = ap.parse_args()
    B = a.batch
    sd, pack = synth.romp_state_dict(0), synth.smpl_pack(0)
    frames = torch.from_numpy(synth.synthetic_frames(B, seed=0)).pin_memory()
    maps, _ = synth.plant_centers(B, seed=0, kmin=1, kmax=10)
    co = torch.from_numpy(maps).cuda()
    res = {}
    outs = {}
    for mode in ("lsq", "epnp"):
        m = ROMP(romp_settings(["--precision", "bf16", "--max_batch", str(B), "--cam_trans", mode]), state_dict=sd, smpl_pack=pack)
        outs[mode] = m.forward_batch(frames, center_override=co)                 # warm-up: graphs, buffers
        ts = []
        for _ in range(a.iters):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            m.forward_batch(frames, center_override=co)
            ts.append(time.perf_counter() - t0)
        res[f"forward_batch_ms_{mode}"] = round(1e3 * float(np.median(ts)), 2)
        if mode == "epnp":
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                for _ in range(a.iters):
                    m.forward_batch(frames, center_override=co)
                torch.cuda.synchronize()
            us = [e.device_time for e in prof.events() if "cam_trans_pnp_kernel" in e.name]
            res["cam_trans_pnp_us_per_batch"] = round(float(np.sum(us)) / max(len(us), 1), 1)
            res["cam_trans_pnp_launches"] = len(us)
        del m
    o = outs["lsq"]
    res["persons"] = int(len(o["cam"]))
    try:
        import cv2  # noqa: F401
        ts = []
        for _ in range(3):
            t0 = time.perf_counter()
            estimate_translation_pnp(o["joints"], o["cam"])
            ts.append(time.perf_counter() - t0)
        res["host_pnp_ms_per_batch"] = round(1e3 * float(np.median(ts)), 1)
    except ImportError:
        res["host_pnp_ms_per_batch"] = None
    name, power = card()
    res.update(batch=B, precision="bf16", gpu=name, power_limit=power, iters=a.iters)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
