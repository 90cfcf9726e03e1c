"""Time BEV's crowd mode on lists of wide images: a loop of process_long_image against one process_long_images call.

    python tools/bev_long_batch_profile.py [--precision bf16] [--max_batch 32] [--warmup 2] [--iters 7]

Lists: 8 and 16 seeded 1080x3840 BGR images (22 crops each), and a mixed list (1080x2160, 1080x3840, 720x2560), every
crop with a planted 3-D centre map (center3d_override) and synthetic weights, as in tools/bev_long_profile.py.  For each
list the two forms run alternately in one process; after warm-up the median of --iters runs of each is reported:
  e2e_ms_per_image    : host wall clock of the call (numpy images in, numpy dicts out) / images
  device_ms_per_image : CUDA events on the BEV stream around the call with device images and to_numpy=False / images
  images_per_s        : images / end-to-end time
The card name and power limit (read-only queries) are printed beside the numbers.
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

from romp_b200 import synth  # noqa: E402
from romp_b200.bev import BEV, bev_settings, long_image_plan  # noqa: E402
from tests import bev_long_oracle as L  # noqa: E402
from tools.bev_long_profile import card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--precision", default="bf16", choices=["bf16", "tf32", "fp32"])
    ap.add_argument("--max_batch", type=int, default=32)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--iters", type=int, default=7)
    a = ap.parse_args()
    s = bev_settings(["--precision", a.precision, "--max_batch", str(a.max_batch)])
    m = BEV(s, state_dict=synth.bev_damp_cam_offsets(synth.bev_state_dict(0)), smpla_pack=synth.smpl_pack(0, num_betas=11),
            smil_pack=synth.smpl_pack(1))
    lists = {"8x1080x3840": [(1080, 3840)] * 8, "16x1080x3840": [(1080, 3840)] * 16,
             "mixed": [(1080, 2160), (1080, 3840), (720, 2560)]}
    name, power = card()
    for label, shapes in lists.items():
        images = [L.long_image(h, w, 100 + i) for i, (h, w) in enumerate(shapes)]
        counts = [len(long_image_plan(h, w, s.overlap_ratio)[1]) for h, w in shapes]
        vols = [torch.from_numpy(L.planted_volumes(k, 200 + i)).cuda() for i, k in enumerate(counts)]
        vall = torch.cat(vols)
        dev = [torch.from_numpy(x).cuda() for x in images]
        torch.cuda.synchronize()
        n = len(images)

        def loop(imgs, to_numpy=True):
            return [m.process_long_image(x, center3d_override=v, to_numpy=to_numpy) for x, v in zip(imgs, vols)]

        def batch(imgs, to_numpy=True):
            return m.process_long_images(imgs, center3d_override=vall, to_numpy=to_numpy)

        def e2e(fn):
            t0 = time.perf_counter()
            fn(images)
            return (time.perf_counter() - t0) * 1e3

        def device(fn):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(m.stream)
            fn(dev, to_numpy=False)
            e1.record(m.stream)
            e1.synchronize()
            return e0.elapsed_time(e1)

        a_out, b_out = loop(images), batch(images)
        equal = all((x is None) == (y is None) and (x is None or all(np.array_equal(x[k], y[k]) for k in x)) for x, y in zip(a_out, b_out))
        times = {k: [] for k in ("loop_e2e", "batch_e2e", "loop_dev", "batch_dev")}
        for it in range(a.warmup + a.iters):
            row = (e2e(loop), e2e(batch), device(loop), device(batch))
            if it >= a.warmup:
                for k, t in zip(times, row):
                    times[k].append(t)
        med = {k: float(np.median(v)) for k, v in times.items()}
        res = {"list": label, "images": n, "crops": sum(counts), "precision": a.precision, "max_batch": m.max_batch,
               "bit_equal": bool(equal), "persons": [0 if x is None else len(x["cam"]) for x in b_out]}
        for form in ("loop", "batch"):
            res[f"{form}_e2e_ms_per_image"] = round(med[f"{form}_e2e"] / n, 3)
            res[f"{form}_device_ms_per_image"] = round(med[f"{form}_dev"] / n, 3)
            res[f"{form}_images_per_s"] = round(1e3 * n / med[f"{form}_e2e"], 2)
        res.update(gpu=name, power_limit=power, iters=a.iters, warmup=a.warmup)
        print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
