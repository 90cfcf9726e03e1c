"""Time the stream mode (--video_streams) of BEV and ROMP against the default video mode on K synthetic cameras.

    python tools/video_streams_profile.py [--cameras 4 16 64] [--ticks 32] [--iters 3] [--precision bf16]

K cameras of 480x640 frames (one random image per camera), --ticks ticks, one list of K frames per tick (camera k is
signal_ID k), through BEV.forward_image_batches and ROMP.forward_video_batches over the whole run.  People are planted
through center3d_override (BEV, up to 12 per camera) and center_override (ROMP, up to 8 per camera); the override applies
to every list, so they stand still, and the trackers still run their full per-frame step on every frame.
Per model and K, for ``streams`` (--video_streams K: one tracker per camera, one CTA per camera) and ``baseline`` (the
default -t mode fed the same lists as one stream, signal_ID 0 for every frame: the serial one-CTA kernel):
  frames_per_s_<mode>       : K * ticks / host wall clock of the whole run, median of --iters runs after one warm-up run;
  track_us_per_batch_<mode> : device time of the track kernels per tick (torch.profiler, a separate run): the step kernel,
                              and in stream mode BEV's row compaction.
The card name and power limit (read-only queries) are printed beside the numbers.  Synthetic weights.
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bev_track_profile import card  # noqa: E402
from romp_b200 import ROMP, romp_settings, synth  # noqa: E402
from romp_b200.bev import BEV, bev_settings  # noqa: E402


def bev_override(K, seed=0):
    """[K,64,128,128]: per camera 12 people at random cells of the 3-D centre map over a low background"""
    rs = np.random.RandomState(seed)
    vol = rs.uniform(0, 0.05, (K, 64, 128, 128)).astype(np.float32)
    for k in range(K):
        for z, y, x in zip(rs.randint(16, 48, 12), rs.randint(8, 120, 12), rs.randint(8, 120, 12)):
            vol[k, z, y, x] = rs.uniform(0.3, 0.9)
    return torch.from_numpy(vol).cuda()


def romp_override(K, seed=0):
    """[K,1,64,64]: per camera 8 people on the centre map"""
    rs = np.random.RandomState(seed)
    maps = np.zeros((K, 1, 64, 64), np.float32)
    for k in range(K):
        for y, x in zip(rs.randint(4, 60, 8), rs.randint(4, 60, 8)):
            maps[k, 0, y, x] = rs.uniform(0.4, 0.9)
    return torch.from_numpy(maps).cuda()


def run(model, lists, sids, override):
    """the whole run on the two-slot pipeline: wall seconds"""
    model.reset_temporal()
    t0 = time.perf_counter()
    if isinstance(model, BEV):
        for _ in model.forward_image_batches(iter(lists), center3d_override=override, signal_IDs=iter(sids)):
            pass
    else:
        for _ in model.forward_video_batches(iter(lists), iter(sids), center_override=override):
            pass
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def track_us_per_batch(model, lists, sids, override):
    """device time of the track kernels per list, from torch.profiler"""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run(model, lists, sids, override)
    us = sum(e.device_time_total for e in prof.key_averages() if "track" in e.key and "kernel" in e.key)
    return round(us / len(lists), 1)


def measure(name, make, override, cameras, ticks, iters):
    rs = np.random.RandomState(1)
    imgs = [rs.randint(0, 256, (480, 640, 3)).astype(np.uint8) for _ in range(max(cameras))]
    models = dict(streams=make(["--video_streams", str(max(cameras))]), baseline=make([]))
    out = []
    for K in cameras:
        lists = [imgs[:K]] * ticks
        res = dict(model=name, cameras=K, ticks=ticks)
        for mode, m in models.items():
            sids = [list(range(K)) if mode == "streams" else [0] * K] * ticks
            ov = override[:K]
            run(m, lists, sids, ov)                                              # warm-up
            ts = [run(m, lists, sids, ov) for _ in range(iters)]
            res[f"frames_per_s_{mode}"] = round(K * ticks / float(np.median(ts)), 1)
            res[f"track_us_per_batch_{mode}"] = track_us_per_batch(m, lists, sids, ov)
        out.append(res)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cameras", type=int, nargs="+", default=[4, 16, 64])
    ap.add_argument("--ticks", type=int, default=32)
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--precision", default="bf16", choices=["bf16", "tf32", "fp32"])
    a = ap.parse_args()
    B = max(a.cameras)
    flags = ["--precision", a.precision, "--max_batch", str(B), "-t"]
    bev_w = dict(state_dict=synth.bev_damp_cam_offsets(synth.bev_state_dict(0)), smpla_pack=synth.smpl_pack(0, num_betas=11),
                 smil_pack=synth.smpl_pack(1))
    romp_w = dict(state_dict=synth.romp_state_dict(0), smpl_pack=synth.smpl_pack(0))
    rows = measure("BEV", lambda x: BEV(bev_settings(flags + x), **bev_w), bev_override(B), a.cameras, a.ticks, a.iters)
    torch.cuda.empty_cache()
    rows += measure("ROMP", lambda x: ROMP(romp_settings(flags + x), **romp_w), romp_override(B), a.cameras, a.ticks, a.iters)
    gpu, power = card()
    for r in rows:
        r.update(precision=a.precision, gpu=gpu, power_limit=power, iters=a.iters)
        print(json.dumps(r))


if __name__ == "__main__":
    main()
