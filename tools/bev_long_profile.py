"""Time BEV's long-image (crowd) mode on one seeded 1080x3840 BGR image (22 crops) with planted 3-D centre maps.

    python tools/bev_long_profile.py [--precision bf16] [--warmup 3] [--iters 10]

Reports, after warm-up, the median of --iters runs of
  end_to_end_ms : BEV.process_long_image(image) (what BEV.forward runs for a wide image), numpy in, dict out, host wall clock
                  ending in the stream sync of the result;
  device_ms     : CUDA events on the BEV stream from the staged device image to the final person count;
  one_by_one_ms : the baseline the batching replaces - the same 22 crops sent one at a time through the normal-image path
                  (host OpenCV img_preprocess + forward_batch at batch 1), host wall clock.
The card name and power limit (read-only queries) are printed beside the numbers.  Weights are synthetic.
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

from romp_b200 import synth  # noqa: E402
from romp_b200.bev import BEV, bev_settings, long_image_plan  # noqa: E402
from romp_b200.main import img_preprocess  # noqa: E402
from tests import bev_long_oracle as L  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [x.strip() for x in q.split(",")]
    except Exception:
        name, power = torch.cuda.get_device_name(0), "unknown"
    return name, power


def median_ms(fn, warmup, iters):
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(iters):
        ts.append(fn())
    return float(np.median(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--precision", default="bf16", choices=["bf16", "tf32", "fp32"])
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--iters", type=int, default=10)
    a = ap.parse_args()
    h, w = 1080, 3840
    s = bev_settings(["--precision", a.precision])
    m = BEV(s, state_dict=synth.bev_damp_cam_offsets(synth.bev_state_dict(0)), smpla_pack=synth.smpl_pack(0, num_betas=11),
            smil_pack=synth.smpl_pack(1))
    image = L.long_image(h, w, 1)
    pad, boxes, _ = long_image_plan(h, w, s.overlap_ratio)
    K = len(boxes)
    vols = torch.from_numpy(L.planted_volumes(K, 2)).cuda()
    torch.cuda.synchronize()
    persons = []

    def end_to_end():
        t0 = time.perf_counter()
        out = m.process_long_image(image, center3d_override=vols)
        persons.append(0 if out is None else len(out["cam"]))
        return (time.perf_counter() - t0) * 1e3

    img_dev = torch.from_numpy(image).cuda()
    torch.cuda.synchronize()

    def device():
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(m.stream)
        m.process_long_image(img_dev, center3d_override=vols, to_numpy=False)
        e1.record(m.stream)
        e1.synchronize()
        return e0.elapsed_time(e1)

    host_pad = np.zeros((h, w + 2 * pad, 3), np.uint8)
    host_pad[:, pad:pad + w] = image
    crops = [np.ascontiguousarray(host_pad[t:b, l:r]) for l, r, t, b in boxes.tolist()]

    def one_by_one():
        t0 = time.perf_counter()
        for i, c in enumerate(crops):
            inp, info = img_preprocess(c)
            m.forward_batch(torch.from_numpy(inp), offsets=info, center3d_override=vols[i:i + 1], img_max_side=float(max(c.shape[:2])))
        return (time.perf_counter() - t0) * 1e3

    res = {"image": f"{h}x{w}", "crops": K, "precision": a.precision, "max_batch": m.max_batch,
           "end_to_end_ms": median_ms(end_to_end, a.warmup, a.iters), "device_ms": median_ms(device, a.warmup, a.iters),
           "one_by_one_ms": median_ms(one_by_one, a.warmup, a.iters), "persons": persons[-1]}
    name, power = card()
    res.update(gpu=name, power_limit=power, iters=a.iters, warmup=a.warmup)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
