"""Time ``--inputs`` (romp_b200/cli.py ``run_inputs``) on K = 1, 4 and 8 copies of a seeded 256-frame 720x1280 video, with
-t and --max_batch 32, for ``romp`` and ``bev``, against K single-input runs one after another.

    python tools/cli_multi_profile.py [--frames 256] [--batch 32] [--ks 1,4,8]

Synthetic weights as in tools/cli_profile.py (ROMP's centre head calibrated; BEV with people planted through the
centre-map hook).  Per model and K it reports, in frames/s over all K x frames:
  inputs_fps     : one run_inputs call on the K copies (--open_inputs K, one stream each), end to end;
  single_fps     : K single-input runs (run_video) one after another, each on a fresh instance: K times one measured
                   run, the copies being identical; build_s, the construction of one instance (conv graphs and weights),
                   which the command pays once per run, is reported apart and not counted in either rate;
  decode_fps     : frame extraction + decoding of the K copies on K threads at once (frame_source), alone;
  device_fps     : the batched entry point alone on decoded frames held in memory, in lists mixing the K streams;
  write_fps      : the shared writer pool (cli.INPUT_WRITERS threads) alone on K x frames of frames and results.
The slowest of decode / device / write bounds inputs_fps.  The host CPU count, card name and power limit (read-only
queries) are printed beside the numbers.
"""
import argparse
import json
import os
import shutil
import sys
import tempfile
import threading
import time
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from cli_profile import card, write_video  # noqa: E402
from oracle import romp_oracle as O  # noqa: E402
from romp_b200 import _lib, cli, graph, synth  # noqa: E402
from romp_b200.bev import BEV, bev_settings  # noqa: E402
from romp_b200.main import ROMP, img_preprocess, romp_settings  # noqa: E402


def release(model):
    """Destroy an instance's conv graphs (library memory the instance does not free) before the next is built."""
    torch.cuda.synchronize()
    for nets in model._nets.values():
        for g in nets:
            if isinstance(g, graph.NetBuilder):
                model.lib.b200romp_net_destroy(g.net)
    model._nets.clear()


def built(model):
    """The instance with its conv graphs for uint8 frames built (they are built on first use otherwise)."""
    model._net(_lib.U8)
    return model


def timed(f):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = f()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, out


def decode_fps(videos, work):
    """frame_source of every video on its own thread at once (extraction + decode, as the readers run them)."""
    n = [0] * len(videos)

    def read(k, v):
        for _ in cli.frame_source(v, os.path.join(work, f"decode{k}"))[0]:
            n[k] += 1

    threads = [threading.Thread(target=read, args=(k, v)) for k, v in enumerate(videos)]
    t0 = time.perf_counter()
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    return sum(n) / (time.perf_counter() - t0)


def profile(name, make, videos, frames, work, prefix, hook, co_list):
    """One model at one K: the rates above."""
    K, T, B = len(videos), len(frames), 32
    r = {}
    build_s, model = timed(lambda: built(make(K)))
    r["build_s"] = round(build_s, 2)
    s, _ = timed(lambda: cli.run_inputs(model, videos, os.path.join(work, f"{name}{K}_inputs"),
                                        types.SimpleNamespace(open_inputs=K, save_video=False, frame_rate=30), prefix, hook))
    r["inputs_fps"] = round(K * T / s, 1)
    release(model)
    one = built(make(0))
    args = types.SimpleNamespace(input=videos[0], save_path=os.path.join(work, f"{name}{K}_single"), save_video=False,
                                 frame_rate=30)
    s, _ = timed(lambda: cli.run_video(one, args, prefix, co_list))
    r["single_fps"] = round(T / s, 1)
    release(one)
    r["decode_fps"] = round(decode_fps(videos, os.path.join(work, f"{name}{K}_decode")), 1)
    model = built(make(K))
    # every K consecutive frames are one frame of each stream: the lists mix the K streams as run_inputs' do
    order = [(k, t) for t in range(T) for k in range(K)]
    lists = [order[i:i + B] for i in range(0, len(order), B)]
    imgs = lambda: ([frames[t] for _, t in lst] for lst in lists)
    sids = lambda: ([k for k, _ in lst] for lst in lists)
    if isinstance(model, ROMP):
        s, res = timed(lambda: sum(model.forward_video_batches(imgs(), sids(), True), []))
    else:
        s, res = timed(lambda: sum(model.forward_image_batches(imgs(), True, co_list, sids()), []))
    r["device_fps"] = round(len(order) / s, 1)
    release(model)
    pool = cli.WriterPool(cli.INPUT_WRITERS)
    savers = [cli.ResultSaver("video", os.path.join(work, f"{name}{K}_write{k}"), pool=pool) for k in range(K)]
    t0 = time.perf_counter()
    for (k, t), o in zip(order, res):
        savers[k](o, f"{t:08d}.jpg", prefix, image=frames[t])
    for sv in savers:
        sv.close()
    r["write_fps"] = round(len(order) / (time.perf_counter() - t0), 1)
    pool.shutdown()
    r["bound_by"] = min(("decode", r["decode_fps"]), ("device", r["device_fps"]), ("write", r["write_fps"]), key=lambda x: x[1])[0]
    print(name, K, json.dumps(r), file=sys.stderr, flush=True)
    for d in [f"_write{k}" for k in range(K)] + ["_inputs", "_single", "_decode"]:
        shutil.rmtree(os.path.join(work, f"{name}{K}{d}"), ignore_errors=True)
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=256)
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--ks", type=str, default="1,4,8")
    a = ap.parse_args()
    ks = [int(k) for k in a.ks.split(",")]
    B = a.batch
    work = tempfile.mkdtemp(prefix="cli_multi_profile_")
    res = {}
    try:
        src = os.path.join(work, "clip.avi")
        write_video(src, a.frames)
        frames = [img for _, img in cli.frame_source(src, os.path.join(work, "frames"))[0]]
        videos = []
        for k in range(max(ks)):
            d = os.path.join(work, f"in{k}")
            os.makedirs(d)
            videos.append(os.path.join(d, f"clip{k}.avi"))
            shutil.copyfile(src, videos[-1])

        sd, pack = synth.romp_state_dict(0), synth.smpl_pack(0)
        rs = np.random.RandomState(1)
        c, _ = O.romp_maps(sd, np.concatenate([img_preprocess(rs.randint(0, 256, (720, 1280, 3)).astype(np.uint8))[0]
                                               for _ in range(2)]))
        sd, _, _ = synth.calibrate_center_head(sd, c.numpy(), max_per_frame=6)
        make = lambda k: ROMP(romp_settings(["--max_batch", str(B), "-t", "--video_streams", str(k)]), state_dict=sd, smpl_pack=pack)
        release(built(make(0)))                                         # warm-up: CUDA context, kernels
        res["romp"] = {k: profile("romp", make, videos[:k], frames, work, None, None, None) for k in ks}

        bsd, smpla, smil = synth.bev_damp_cam_offsets(synth.bev_state_dict(0)), synth.smpl_pack(0, num_betas=11), synth.smpl_pack(1)
        vol, _ = synth.plant_centers_3d(B, seed=2)
        co = torch.from_numpy(vol).cuda()
        hook = lambda i, t: co[t % B]
        make = lambda k: BEV(bev_settings(["--max_batch", str(B), "-t", "--video_streams", str(k)]), state_dict=bsd,
                             smpla_pack=smpla, smil_pack=smil)
        s = bev_settings([])
        res["bev"] = {k: profile("bev", make, videos[:k], frames, work, f"_2_{s.center_thresh}", hook, co) for k in ks}
    finally:
        shutil.rmtree(work, ignore_errors=True)
    name, power = card()
    res.update(frames=a.frames, batch=B, image="720x1280", writers=cli.INPUT_WRITERS, precision="bf16", cpus=os.cpu_count(),
               gpu=name, power_limit=power)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
