"""Time the ``romp`` and ``bev`` video modes (romp_b200/cli.py) on a seeded 256-frame 720x1280 video, both with -t,
against the reference's per-frame loop, and check that both write identical files.

    python tools/cli_profile.py [--frames 256] [--batch 32] [--writers 4]

Synthetic weights: ROMP's centre head calibrated to a few people per frame; BEV with people planted through the 3-D
centre-map override.  For each model it reports, in frames/s:
  cli_fps        : cli.run_video end to end (frame extraction + decode on the reader thread, the batched GPU path,
                   PNG / npz writers), then video_results.npz;
  loop_fps       : the reference's loop: extract every frame to disk, then per frame cv2.imread, one single-frame call of
                   the same GPU path (so that every file is identical) and a serial ResultSaver; then video_results.npz;
  decode_fps     : extraction + in-memory decode alone (frame_source);
  device_fps     : the batched entry point alone on the decoded frames (held in memory);
  write_fps      : the writer pool alone on those frames and results.
The slowest of decode / device / write bounds cli_fps.  The card name and power limit (read-only queries) are printed
beside the numbers.
"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time
import types

import cv2
import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import romp_oracle as O  # noqa: E402
from romp_b200 import cli, synth  # noqa: E402
from romp_b200.bev import BEV, bev_settings  # noqa: E402
from romp_b200.main import ROMP, img_preprocess, romp_settings  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [x.strip() for x in q.split(",")]
    except Exception:
        name, power = torch.cuda.get_device_name(0), "unknown"
    return name, power


def write_video(path, T, h=720, w=1280, seed=0):
    rs = np.random.RandomState(seed)
    base = rs.randint(0, 256, (h, w, 3)).astype(np.int16)
    vw = cv2.VideoWriter(path, cv2.VideoWriter_fourcc(*"MJPG"), 30, (w, h))
    for t in range(T):
        f = np.clip(base + rs.randint(-6, 7, base.shape), 0, 255).astype(np.uint8)
        f[200:400, (7 * t) % (w - 200):(7 * t) % (w - 200) + 200] = 220
        vw.write(f)
    vw.release()


def same_value(a, b, where):
    if isinstance(a, dict):
        assert isinstance(b, dict) and list(a) == list(b), where
        for k in a:
            same_value(a[k], b[k], where)
    elif isinstance(a, list):
        assert isinstance(b, list) and len(a) == len(b), where
        for x, y in zip(a, b):
            same_value(x, y, where)
    else:
        x, y = np.asarray(a), np.asarray(b)
        assert x.dtype == y.dtype and x.shape == y.shape and np.array_equal(x, y), where


def same_files(d1, d2):
    names = sorted(os.listdir(d1))
    assert names == sorted(os.listdir(d2)), "different file sets"
    for n in names:
        a, b = os.path.join(d1, n), os.path.join(d2, n)
        if os.path.isdir(a):
            continue
        if n.endswith(".npz"):
            x, y = np.load(a, allow_pickle=True), np.load(b, allow_pickle=True)
            for k in x.files:
                same_value(x[k][()], y[k][()], n)
        else:
            with open(a, "rb") as f, open(b, "rb") as g:
                assert f.read() == g.read(), n
    return len(names)


def profile(name, make, one, video, work, prefix, override, writers):
    T = int(cv2.VideoCapture(video).get(cv2.CAP_PROP_FRAME_COUNT))
    r = {}
    # warm-up: graphs and staging buffers of both paths
    warm = make()
    cli.run_frames(warm, [(f"w{i}.jpg", np.zeros((720, 1280, 3), np.uint8)) for i in range(4)],
                   cli.ResultSaver("video", os.path.join(work, "warm")), prefix, override)
    del warm

    out_cli = os.path.join(work, name + "_cli")
    args = types.SimpleNamespace(input=video, save_path=out_cli, save_video=False, frame_rate=30)
    model = make()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    cli.run_video(model, args, prefix, override)
    r["cli_fps"] = round(T / (time.perf_counter() - t0), 1)
    del model

    out_loop = os.path.join(work, name + "_loop")
    model = make()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    paths, _ = cli.collect_frame_path(video, out_loop)
    saver = cli.ResultSaver("video", out_loop)
    for i, p in enumerate(paths):
        saver(one(model, cv2.imread(p), i), p, prefix)
    cli.save_video_results(saver.frame_save_paths)
    r["loop_fps"] = round(T / (time.perf_counter() - t0), 1)
    del model
    r["files_compared"] = same_files(out_cli, out_loop)

    t0 = time.perf_counter()
    frames = list(cli.frame_source(video, os.path.join(work, name + "_decode"))[0])
    r["decode_fps"] = round(T / (time.perf_counter() - t0), 1)
    model = make()
    lists = [[img for _, img in frames[i:i + model.max_batch]] for i in range(0, T, model.max_batch)]
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    if isinstance(model, ROMP):
        res = sum(model.forward_video_batches(iter(lists), None, True, override), [])
    else:
        res = sum(model.forward_image_batches(iter(lists), True, override), [])
    r["device_fps"] = round(T / (time.perf_counter() - t0), 1)
    del model
    saver = cli.ResultSaver("video", os.path.join(work, name + "_write"), writers=writers)
    t0 = time.perf_counter()
    for (p, img), o in zip(frames, res):
        saver(o, p, prefix, image=img)
    saver.close()
    r["write_fps"] = round(T / (time.perf_counter() - t0), 1)
    r["people_per_frame"] = round(float(np.mean([0 if o is None else len(o["cam"]) for o in res])), 2)
    r["bound_by"] = min(("decode", r["decode_fps"]), ("device", r["device_fps"]), ("write", r["write_fps"]), key=lambda x: x[1])[0]
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=256)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--writers", type=int, default=cli.WRITERS)
    a = ap.parse_args()
    cli.WRITERS = a.writers
    work = tempfile.mkdtemp(prefix="cli_profile_")
    try:
        video = os.path.join(work, "clip.avi")
        write_video(video, a.frames)
        B = a.batch
        sd, pack = synth.romp_state_dict(0), synth.smpl_pack(0)
        rs = np.random.RandomState(1)
        c, _ = O.romp_maps(sd, np.concatenate([img_preprocess(rs.randint(0, 256, (720, 1280, 3)).astype(np.uint8))[0]
                                               for _ in range(2)]))
        sd, _, _ = synth.calibrate_center_head(sd, c.numpy(), max_per_frame=6)
        res = {}
        make = lambda: ROMP(romp_settings(["--max_batch", str(B), "-t"]), state_dict=sd, smpl_pack=pack)
        res["romp"] = profile("romp", make, lambda m, img, i: m.forward_video([img])[0], video, work, None, None, a.writers)

        bsd, smpla, smil = synth.bev_damp_cam_offsets(synth.bev_state_dict(0)), synth.smpl_pack(0, num_betas=11), synth.smpl_pack(1)
        vol, _ = synth.plant_centers_3d(B, seed=2)
        co = torch.from_numpy(vol).cuda()
        s = bev_settings(["--max_batch", str(B), "-t"])
        make = lambda: BEV(s, state_dict=bsd, smpla_pack=smpla, smil_pack=smil)
        res["bev"] = profile("bev", make, lambda m, img, i: m.forward_images([img], center3d_override=co[i % B:i % B + 1])[0],
                             video, work, f"_2_{s.center_thresh}", co, a.writers)
    finally:
        shutil.rmtree(work, ignore_errors=True)
    name, power = card()
    res.update(frames=a.frames, batch=B, image="720x1280", writers=a.writers, precision="bf16", cpus=os.cpu_count(), gpu=name,
               power_limit=power)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
