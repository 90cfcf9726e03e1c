"""Time BEV's video mode (-t) on a seeded synthetic video: 256 frames, 10-30 moving people planted through
center3d_override, synthetic weights.

    python tools/bev_track_profile.py [--precision bf16] [--batch 32] [--iters 3]

Reports (median of --iters runs after one warm-up run of each):
  frames_per_s_t        : BEV.forward_images(frames, center3d_override=...) with -t, in chunks of --batch frames (numpy in,
                          per-frame dicts out; host wall clock, each chunk ends in its stream sync);
  frames_per_s_plain    : the same call on an instance without -t;
  track_kernel_us_per_frame : CUDA events on the BEV stream around b200romp_bev_track_step, summed over the video / frames;
  oracle_cpu_us_per_frame  : CPU figure, for context: oracle/track_oracle.py (numpy, the reference's algorithm) stepping
                          the same video's parse outputs on the host;
  extra_device_mb       : device memory a -t instance allocates beyond a plain one at this --batch.
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

from oracle import track_oracle as TO  # noqa: E402
from romp_b200 import synth  # noqa: E402
from romp_b200.bev import BEV, bev_settings  # noqa: E402
from romp_b200.main import img_preprocess  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [x.strip() for x in q.split(",")]
    except Exception:
        name, power = torch.cuda.get_device_name(0), "unknown"
    return name, power


def trajectories(T, seed):
    """Per frame, the planted cells (z, y, x, value) of 10-30 people walking, entering and leaving."""
    rs = np.random.RandomState(seed)
    people = []
    for _ in range(40):
        t0 = int(rs.randint(0, T // 2)) if len(people) >= 12 else 0
        people.append(dict(t0=t0, t1=int(rs.randint(t0 + 60, T + 60)), p=np.array([rs.uniform(20, 44), rs.uniform(8, 120), rs.uniform(8, 120)]),
                           v=np.array([0.0, rs.uniform(-0.3, 0.3), rs.uniform(-0.3, 0.3)]), val=rs.uniform(0.3, 0.9)))
    frames = []
    for t in range(T):
        cells = []
        for q in people:
            q["p"] = q["p"] + q["v"]
            for a in (1, 2):
                if not 8 <= q["p"][a] <= 120:
                    q["v"][a] = -q["v"][a]
            if not q["t0"] <= t < q["t1"] or len(cells) >= 30:
                continue
            z, y, x = (int(round(c)) for c in q["p"])
            if all(max(abs(z - c[0]), abs(y - c[1]), abs(x - c[2])) >= 3 for c in cells):
                cells.append((z, y, x, q["val"]))
        frames.append(cells)
    return frames


def volumes(cells, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    vol = torch.rand((len(cells), 64, 128, 128), generator=g, device="cuda") * 0.05
    for b, cs in enumerate(cells):
        for z, y, x, v in cs:
            vol[b, z, y, x] = v
    return vol


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--precision", default="bf16", choices=["bf16", "tf32", "fp32"])
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--frames", type=int, default=256)
    ap.add_argument("--iters", type=int, default=3)
    a = ap.parse_args()
    T, B = a.frames, a.batch
    params = dict(state_dict=synth.bev_damp_cam_offsets(synth.bev_state_dict(0)), smpla_pack=synth.smpl_pack(0, num_betas=11),
                  smil_pack=synth.smpl_pack(1))
    cells = trajectories(T, 0)
    counts = [len(c) for c in cells]
    img = np.random.RandomState(1).randint(0, 256, (480, 640, 3)).astype(np.uint8)
    imgs = [img] * T
    vols = [volumes(cells[c0:c0 + B], c0) for c0 in range(0, T, B)]
    flags = ["--precision", a.precision, "--max_batch", str(B)]
    torch.cuda.synchronize()
    m0 = torch.cuda.memory_allocated()
    plain = BEV(bev_settings(flags), **params)
    m1 = torch.cuda.memory_allocated()
    tm = BEV(bev_settings(flags + ["-t"]), **params)
    m2 = torch.cuda.memory_allocated()

    # the track kernel's device time: CUDA events on the BEV stream around every step
    spans = []
    run_temporal = tm.run_temporal

    def timed_run_temporal(*args):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(tm.stream)
        run_temporal(*args)
        e1.record(tm.stream)
        spans.append((e0, e1))
    tm.run_temporal = timed_run_temporal

    def video(m):
        if m is tm:
            m.reset_temporal()
        out, t0 = [], time.perf_counter()
        for k, c0 in enumerate(range(0, T, B)):
            out += m.forward_images(imgs[c0:c0 + B], center3d_override=vols[k])
        return time.perf_counter() - t0, out

    res = {}
    for name, m in (("plain", plain), ("t", tm)):
        video(m)                                                             # warm-up: graphs, staging buffers
        ts, kern = [], []
        for _ in range(a.iters):
            spans.clear()
            dt, out = video(m)
            ts.append(dt)
            if m is tm:
                torch.cuda.synchronize()
                kern.append(sum(e0.elapsed_time(e1) for e0, e1 in spans) * 1e3 / T)
        res[f"frames_per_s_{name}"] = round(T / float(np.median(ts)), 1)
        if m is tm:
            res["track_kernel_us_per_frame"] = round(float(np.median(kern)), 2)
            res["rows_out"] = int(sum(0 if o is None else len(o["track_ids"]) for o in out))
            res["ids"] = int(len({i for o in out if o is not None for i in o["track_ids"].tolist()}))

    # CPU figure: the oracle tracker on the same parse outputs (read from a plain instance's device rows)
    parsed = []
    for k, c0 in enumerate(range(0, T, B)):
        nb = min(B, T - c0)
        frames = torch.from_numpy(np.ascontiguousarray(np.repeat(img_preprocess(img)[0], nb, 0))).cuda()
        with torch.cuda.stream(plain.stream):
            plain.run_model(frames, vols[k])
        plain.stream.synchronize()
        n = int(plain.buf["count"].item())
        b = {key: plain.buf[src][:n].cpu().numpy() for key, src in (("smpl_thetas", "thetas"), ("smpl_betas", "betas"), ("cam", "cam"),
                                                                     ("cam_trans", "cam_trans"), ("params_pred", "params_pred"),
                                                                     ("center_confs", "conf"), ("pred_batch_ids", "batch_ids"))}
        for f in range(nb):
            sel = b["pred_batch_ids"] == f
            parsed.append({key: v[sel] for key, v in b.items()} if sel.any() else {})
    host = []
    for _ in range(a.iters):
        sm = TO.TemporalBEV()
        t0 = time.perf_counter()
        for f in parsed:
            if f:
                sm(f, 0)
        host.append((time.perf_counter() - t0) * 1e6 / T)
    res["oracle_cpu_us_per_frame"] = round(float(np.median(host)), 1)
    name, power = card()
    res.update(people_per_frame=[min(counts), max(counts)], frames=T, batch=B, precision=a.precision,
               extra_device_mb=round(((m2 - m1) - (m1 - m0)) / 2**20, 1), gpu=name, power_limit=power, iters=a.iters)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
