"""Time ROMP's video mode (-t) on a seeded synthetic video: 256 frames of 480x640 BGR images (a scene with small
frame-to-frame changes), synthetic weights with the center head calibrated to a few people per frame.

    python tools/romp_video_profile.py [--precision bf16] [--batch 32] [--frames 256] [--iters 3] [--modes tracked,largest]

Reports, for the tracked mode and for --show_largest (median of --iters runs after one warm-up run of each; host wall
clock, numpy images in, per-frame dicts out):
  video_fps            : ROMP.forward_video(images) in chunks of --batch frames;
  images_fps_plain     : ROMP.forward_images(images) on an instance without -t (no tracking, no smoothing);
  forward_loop_fps     : [ROMP.forward(img) for img in images] with -t, the per-frame path;
  track_step_us_per_batch : device time of the track step kernel (b200romp_romp_track_step) per chunk, from
                         torch.profiler in a separate run of forward_video.
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

from oracle import romp_oracle as O  # noqa: E402
from romp_b200 import ROMP, romp_settings, synth  # noqa: E402
from romp_b200.main import img_preprocess  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [x.strip() for x in q.split(",")]
    except Exception:
        name, power = torch.cuda.get_device_name(0), "unknown"
    return name, power


def video(T, seed=0):
    rs = np.random.RandomState(seed)
    base = rs.randint(0, 256, (480, 640, 3)).astype(np.int16)
    return [np.clip(base + rs.randint(-6, 7, base.shape), 0, 255).astype(np.uint8) for _ in range(T)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--precision", default="bf16", choices=["bf16", "tf32", "fp32"])
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--frames", type=int, default=256)
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--modes", default="tracked,largest", help="video modes to time, in this order")
    a = ap.parse_args()
    T, B = a.frames, a.batch
    imgs = video(T)
    sd, pack = synth.romp_state_dict(0), synth.smpl_pack(0)
    c, _ = O.romp_maps(sd, np.concatenate([img_preprocess(x)[0] for x in imgs[:4]]))
    sd, _, _ = synth.calibrate_center_head(sd, c.numpy(), max_per_frame=6)
    flags = ["--precision", a.precision, "--max_batch", str(B)]
    make = lambda extra: ROMP(romp_settings(flags + extra), state_dict=sd, smpl_pack=pack)

    def timed(fn, reset=None):
        fn()                                                                 # warm-up: graphs, staging buffers
        ts = []
        for _ in range(a.iters):
            if reset is not None:
                reset()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            out = fn()
            ts.append(time.perf_counter() - t0)
        return round(T / float(np.median(ts)), 1), out

    res = {}
    plain = make([])
    res["images_fps_plain"], out = timed(lambda: plain.forward_images(imgs))
    res["people_per_frame"] = [min(0 if o is None else len(o["cam"]) for o in out), max(0 if o is None else len(o["cam"]) for o in out)]
    del plain
    for mode in a.modes.split(","):
        extra = {"tracked": ["-t"], "largest": ["-t", "--show_largest"]}[mode]
        m = make(extra)
        r = {}
        r["video_fps"], _ = timed(lambda: m.forward_video(imgs), m.reset_temporal)
        m.reset_temporal()
        r["forward_loop_fps"], _ = timed(lambda: [m.forward(x) for x in imgs], m.reset_temporal)
        m.reset_temporal()
        m.forward_video(imgs)                                                # warm
        m.reset_temporal()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            m.forward_video(imgs)
            torch.cuda.synchronize()
        us = [e.device_time for e in prof.events() if "romp_track_kernel" in e.name]
        r["track_step_us_per_batch"] = round(float(np.sum(us)) / max(len(us), 1), 1)
        r["track_step_launches"] = len(us)
        res[mode] = r
        del m
    name, power = card()
    res.update(frames=T, batch=B, image="480x640", precision=a.precision, gpu=name, power_limit=power, iters=a.iters)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
