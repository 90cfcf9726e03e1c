"""Time the command lines' video frame extraction (romp_b200/cli.py) with the JPEG round trip on the CPU (cv2, the
``frame_source`` path) and on the GPU (romp_b200.jpeg.FrameCodec), on the seeded 256-frame 720x1280 video of
tools/cli_profile.py, and check that both write identical files.

    python tools/frame_extract_profile.py [--frames 256] [--batch 32] [--rounds 2]

Reports, in frames/s unless named otherwise:
  reader_cpu_fps / reader_gpu_fps : the reader thread's work alone (VideoCapture, JPEG encode, file write, decode)
  codec_ms_per_list               : device time of the codec's kernels per list of --batch frames (torch.profiler, a run
                                    of its own)
  <model>_cpu_fps / _gpu_fps      : cli.run_video end to end with -t, the two extractions alternating for --rounds
                                    rounds in one process; every file compared between the two
The card name and power limit (read-only queries) are printed beside the numbers.
"""
import argparse
import json
import os
import shutil
import sys
import tempfile
import time
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from cli_profile import card, same_files, write_video  # noqa: E402
from oracle import romp_oracle as O  # noqa: E402
from romp_b200 import cli, jpeg, synth  # noqa: E402
from romp_b200.bev import BEV, bev_settings  # noqa: E402
from romp_b200.main import ROMP, img_preprocess, romp_settings  # noqa: E402


def reader_fps(frames_iter):
    t = time.perf_counter()
    n = sum(1 for _ in frames_iter)
    return n / (time.perf_counter() - t)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=256)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--rounds", type=int, default=2)
    a = ap.parse_args()
    B = a.batch
    work = tempfile.mkdtemp(prefix="frame_extract_profile_")
    res = {}
    try:
        video = os.path.join(work, "clip.avi")
        write_video(video, a.frames)
        codec = jpeg.FrameCodec("cuda:0")
        assert codec.usable, codec.reason
        reader_fps(cli.frame_source(video, os.path.join(work, "warm"))[0])
        res["reader_cpu_fps"] = reader_fps(cli.frame_source(video, os.path.join(work, "r_cpu"))[0])
        os.makedirs(os.path.join(work, "r_gpu"))
        list(cli._extract_gpu(codec, video, os.path.join(work, "r_gpu"), B))
        res["reader_gpu_fps"] = reader_fps(cli._extract_gpu(codec, video, os.path.join(work, "r_gpu"), B))
        assert same_files(os.path.join(work, "r_cpu", "clip_frames"), os.path.join(work, "r_gpu")) == a.frames

        import cv2
        cap, frames = cv2.VideoCapture(video), []
        while len(frames) < B:
            frames.append(cap.read()[1])
        cap.release()
        codec.run(frames)
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(5):
                codec.run(frames)
        us = sum(e.device_time_total for e in prof.key_averages() if "jpeg_" in e.key)
        res["codec_ms_per_list"] = us / 5 / 1000.0
        res["codec_kernels"] = sorted({e.key for e in prof.key_averages() if "jpeg_" in e.key})

        sd, pack = synth.romp_state_dict(0), synth.smpl_pack(0)
        rs = np.random.RandomState(1)
        c, _ = O.romp_maps(sd, np.concatenate([img_preprocess(rs.randint(0, 256, (720, 1280, 3)).astype(np.uint8))[0]
                                               for _ in range(2)]))
        sd, _, _ = synth.calibrate_center_head(sd, c.numpy(), max_per_frame=6)
        bsd, smpla, smil = synth.bev_damp_cam_offsets(synth.bev_state_dict(0)), synth.smpl_pack(0, num_betas=11), synth.smpl_pack(1)
        vol, _ = synth.plant_centers_3d(B, seed=2)
        co = torch.from_numpy(vol).cuda()
        bs = bev_settings(["--max_batch", str(B), "-t"])
        models = {"romp": (lambda: ROMP(romp_settings(["--max_batch", str(B), "-t"]), state_dict=sd, smpl_pack=pack), None, None),
                  "bev": (lambda: BEV(bs, state_dict=bsd, smpla_pack=smpla, smil_pack=smil), f"_2_{bs.center_thresh}", co)}
        real_codec = cli.frame_codec
        for name, (make, prefix, override) in models.items():
            times = {"cpu": [], "gpu": []}
            for r in range(a.rounds):
                for path in ("gpu", "cpu"):
                    cli.frame_codec = real_codec if path == "gpu" else (lambda model: None)
                    model = make()
                    out = os.path.join(work, f"{name}_{path}_{r}")
                    args = types.SimpleNamespace(input=video, save_path=out, save_video=False, frame_rate=24)
                    torch.cuda.synchronize()
                    t = time.perf_counter()
                    cli.run_video(model, args, prefix, override)
                    times[path].append(a.frames / (time.perf_counter() - t))
                    del model
            cli.frame_codec = real_codec
            for r in range(a.rounds):
                same_files(os.path.join(work, f"{name}_gpu_{r}"), os.path.join(work, f"{name}_cpu_{r}"))
                same_files(os.path.join(work, f"{name}_gpu_{r}", "clip_frames"), os.path.join(work, f"{name}_cpu_{r}", "clip_frames"))
            res[f"{name}_gpu_fps"] = times["gpu"]
            res[f"{name}_cpu_fps"] = times["cpu"]
        res["files_identical"] = True
    finally:
        shutil.rmtree(work, ignore_errors=True)
    name, power = card()
    res.update(frames=a.frames, batch=B, image="720x1280", cpus=os.cpu_count(), gpu=name, power_limit=power)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
