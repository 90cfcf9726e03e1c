"""Time ROMP on raw images of mixed sizes: the batched image path against the one-image loop.

    python tools/image_batch_profile.py [--precision bf16] [--warmup 2] [--iters 5] [--stream_batches 10]

Images: a seeded mix of 64 BGR images, 16 each of 1080x1920, 720x1280, 1920x1080 (portrait) and 480x640.  Weights are
synthetic, with the center head calibrated to detect (synth.calibrate_center_head).  Reports, after warm-up, medians of
--iters runs of
  per_image_ms        : [ROMP.forward(img) for img in images], host wall clock (each call ends in its own host sync);
  forward_images_ms   : ROMP.forward_images(images), numpy in, lists out, host wall clock ending in the last read-back;
  stream_images_per_s : ROMP.forward_image_batches over --stream_batches lists of the 64 images;
  device_ms           : CUDA events on the model stream from the raw images in device memory to the end of the batch
                        (batched preprocessing, model, parse, SMPL, projection);
  host_staging_ms     : the copy of the 64 images into the pinned staging buffer;
  preprocess_us       : the batched preprocessing kernel on the 64 device images, against 64 single-image launches.
It first asserts that forward_images returns exactly the per-image results.  The card name and power limit (read-only
queries) are printed beside the numbers.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import preproc_oracle as P  # noqa: E402
from oracle import romp_oracle as O  # noqa: E402
from romp_b200 import ROMP, _lib, romp_settings, synth  # noqa: E402
from romp_b200.staging import image_tensor, preprocess_bgr_batch, stage_host_images, staging_layout  # noqa: E402

SHAPES = [(1080, 1920), (720, 1280), (1920, 1080), (480, 640)]


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [x.strip() for x in q.split(",")]
    except Exception:
        name, power = torch.cuda.get_device_name(0), "unknown"
    return name, power


def mixed_images(seed=0):
    rs = np.random.RandomState(seed)
    shapes = [s for s in SHAPES for _ in range(16)]
    order = rs.permutation(len(shapes))
    return [rs.randint(0, 256, (*shapes[i], 3)).astype(np.uint8) for i in order]


def median(fn, warmup, iters):
    for _ in range(warmup):
        fn()
    return float(np.median([fn() for _ in range(iters)]))


def wall(fn):
    def run():
        t = time.perf_counter()
        fn()
        return (time.perf_counter() - t) * 1e3
    return run


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--precision", default="bf16", choices=["bf16", "tf32", "fp32"])
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--stream_batches", type=int, default=10)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "image_batch_profile needs a GPU"
    images = mixed_images()
    sd, pack = synth.romp_state_dict(0), synth.smpl_pack(0)
    calib = np.concatenate([P.img_preprocess(images[i], 512)[0] for i in range(0, 64, 8)])
    sd, _, _ = synth.calibrate_center_head(sd, O.romp_maps(sd, calib)[0].numpy(), max_per_frame=6)
    m = ROMP(romp_settings(["--precision", a.precision, "--max_batch", "64"]), state_dict=sd, smpl_pack=pack)

    # results first: the batched path returns exactly the per-image results
    ref = [m(img) for img in images]
    got = m.forward_images(images)
    persons = 0
    for i, (x, y) in enumerate(zip(got, ref)):
        assert (x is None) == (y is None), f"image {i}"
        if x is not None:
            assert set(x) == set(y) and all(np.array_equal(x[k], y[k]) for k in x), f"image {i}"
            persons += len(x["cam"])
    res = dict(images=len(images), persons=persons, precision=a.precision, results_equal=True)

    res["per_image_ms"] = median(wall(lambda: [m(img) for img in images]), a.warmup, a.iters)
    res["forward_images_ms"] = median(wall(lambda: m.forward_images(images)), a.warmup, a.iters)

    def stream():
        t = time.perf_counter()
        n = sum(len(r) for r in m.forward_image_batches(images for _ in range(a.stream_batches)))
        return n / (time.perf_counter() - t)
    res["stream_images_per_s"] = median(stream, 1, a.iters)

    dev = [torch.from_numpy(x).cuda() for x in images]
    torch.cuda.synchronize()

    def device():
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(m.stream)
        m._submit_images([image_tensor(t) for t in dev], None)
        e1.record(m.stream)
        e1.synchronize()
        return e0.elapsed_time(e1)
    res["device_ms"] = median(device, a.warmup, a.iters)

    host = [torch.from_numpy(x) for x in images]
    offs, total = staging_layout(host)
    pinned = torch.empty(total, dtype=torch.uint8).pin_memory()
    res["host_staging_ms"] = median(wall(lambda: stage_host_images(host, offs, pinned)), a.warmup, a.iters)
    res["raw_mbytes"] = round(total / 1e6, 1)

    out = torch.empty((64, 512, 512, 3), dtype=torch.uint8, device="cuda")
    pad = torch.empty((64, 6), device="cuda")
    s = torch.cuda.current_stream()
    lib = m.lib

    def kernel_us(fn, reps=10):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        fn()
        e0.record(s)
        for _ in range(reps):
            fn()
        e1.record(s)
        e1.synchronize()
        return e0.elapsed_time(e1) * 1e3 / reps

    def singles():
        for i, t in enumerate(dev):
            _lib.check(lib.b200romp_preprocess_bgr(C.c_void_p(t.data_ptr()), t.shape[0], t.shape[1], 3 * t.shape[1], 512,
                                                   C.c_void_p(out[i].data_ptr()), None, C.c_void_p(s.cuda_stream)))
    res["preprocess_us"] = {
        "batched": median(lambda: kernel_us(lambda: preprocess_bgr_batch(lib, dev, [None] * 64, None, out, pad, s.cuda_stream)),
                          1, a.iters),
        "single_launches": median(lambda: kernel_us(singles), 1, a.iters)}
    name, power = card()
    res.update(gpu=name, power_limit=power, iters=a.iters, warmup=a.warmup)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
