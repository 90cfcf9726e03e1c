"""Time BEV's image path and video mode (-t) on a seeded synthetic video: 256 frames, 10-30 moving people planted through
center3d_override, synthetic weights.

    python tools/bev_track_profile.py [--precision bf16] [--batch 32] [--iters 3]

Reports (median of --iters runs after one warm-up run of each), for an instance without -t (``plain``) and one with it (``t``):
  frames_per_s_<m>       : BEV.forward_images(chunk, center3d_override=...) called once per chunk of --batch frames (numpy in,
                           per-frame dicts out; host wall clock), each call ending in its own read-back;
  frames_per_s_<m>_stream: BEV.forward_image_batches([frames]) over the whole video: the same chunks on the two-slot pipeline,
                           staging and read-back of neighbouring chunks overlapping each chunk's kernels;
  device_ms_per_chunk_<m>: CUDA events on the BEV stream from each chunk's run_model to the end of its run_post (the chunk's
                           device work after the preprocessing kernel), median over the chunk loop's chunks;
  wall_ms_per_chunk_<m>[_stream]: host wall clock per chunk of the two calls above;
  track_kernel_us_per_frame : CUDA events on the BEV stream around b200romp_bev_track_step, summed over the video / frames;
  oracle_cpu_us_per_frame  : CPU figure, for context: oracle/track_oracle.py (numpy, the reference's algorithm) stepping
                           the same video's parse outputs on the host;
  extra_device_mb        : device memory a -t instance allocates beyond a plain one at this --batch.
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


def instrument(m):
    """CUDA events on m.stream: from each chunk's run_model to the end of its run_post, and around every track step."""
    spans = dict(chunk=[], track=[])

    def wrap(name, opens, closes):
        f = getattr(m, name)

        def timed(*args, **kw):
            if opens:
                spans[opens].append([torch.cuda.Event(enable_timing=True), None])
                spans[opens][-1][0].record(m.stream)
            r = f(*args, **kw)
            if closes:
                spans[closes][-1][1] = torch.cuda.Event(enable_timing=True)
                spans[closes][-1][1].record(m.stream)
            return r
        setattr(m, name, timed)
    wrap("run_model", "chunk", None)
    wrap("run_post", None, "chunk")
    if m.temporal:
        wrap("run_temporal", "track", "track")
    return spans


def elapsed_ms(spans):
    torch.cuda.synchronize()
    return [e0.elapsed_time(e1) for e0, e1 in spans]


class Video:
    """The seeded 256-frame video and the two ways of running it through a BEV instance."""

    def __init__(self, T, B):
        self.T, self.B = T, B
        self.cells = trajectories(T, 0)
        img = np.random.RandomState(1).randint(0, 256, (480, 640, 3)).astype(np.uint8)
        self.img, self.imgs = img, [img] * T
        self.vol = torch.cat([volumes(self.cells[c0:c0 + B], c0) for c0 in range(0, T, B)])

    def loop(self, m):
        """forward_images once per chunk: wall seconds, per-frame results"""
        if m.temporal:
            m.reset_temporal()
        out, t0 = [], time.perf_counter()
        for c0 in range(0, self.T, self.B):
            out += m.forward_images(self.imgs[c0:c0 + self.B], center3d_override=self.vol[c0:c0 + self.B])
        return time.perf_counter() - t0, out

    def stream(self, m):
        """forward_image_batches over the whole video as one list (the same chunks, pipelined)"""
        if m.temporal:
            m.reset_temporal()
        t0 = time.perf_counter()
        out = next(m.forward_image_batches([self.imgs], center3d_override=self.vol))
        return time.perf_counter() - t0, out


def measure(v, m, name, iters, res, stream=True):
    """frame rates, wall and device time per chunk of instance m into res (keys suffixed with name)"""
    spans = instrument(m)
    chunks = -(-v.T // v.B)
    for how in ("loop", "stream") if stream else ("loop",):
        run = getattr(v, how)
        run(m)                                                               # warm-up: graphs, staging buffers, mirrors
        ts, dev, kern = [], [], []
        for _ in range(iters):
            spans["chunk"].clear()
            spans["track"].clear()
            dt, out = run(m)
            ts.append(dt)
            dev += elapsed_ms(spans["chunk"])
            kern.append(sum(elapsed_ms(spans["track"])) * 1e3 / v.T)
        sfx = name if how == "loop" else name + "_stream"
        res[f"frames_per_s_{sfx}"] = round(v.T / float(np.median(ts)), 1)
        res[f"wall_ms_per_chunk_{sfx}"] = round(float(np.median(ts)) * 1e3 / chunks, 2)
        res[f"device_ms_per_chunk_{sfx}"] = round(float(np.median(dev)), 2)
        if m.temporal and how == "loop":
            res["track_kernel_us_per_frame"] = round(float(np.median(kern)), 2)
            res["rows_out"] = int(sum(0 if o is None else len(o["track_ids"]) for o in out))
            res["ids"] = int(len({i for o in out if o is not None for i in o["track_ids"].tolist()}))
    return spans


def oracle_cpu_us_per_frame(v, plain, iters):
    """The oracle tracker on the video's parse outputs (read from a plain instance's device rows), host time per frame."""
    parsed = []
    T, B = v.T, v.B
    for c0 in range(0, T, B):
        nb = min(B, T - c0)
        frames = torch.from_numpy(np.ascontiguousarray(np.repeat(img_preprocess(v.img)[0], nb, 0))).cuda()
        with torch.cuda.stream(plain.stream):
            plain.run_model(frames, v.vol[c0:c0 + nb])
        plain.stream.synchronize()
        n = int(plain.buf["count"].item())
        b = {key: plain.buf[src][:n].cpu().numpy() for key, src in (("smpl_thetas", "thetas"), ("smpl_betas", "betas"), ("cam", "cam"),
                                                                     ("cam_trans", "cam_trans"), ("params_pred", "params_pred"),
                                                                     ("center_confs", "conf"), ("pred_batch_ids", "batch_ids"))}
        for f in range(nb):
            sel = b["pred_batch_ids"] == f
            parsed.append({key: x[sel] for key, x in b.items()} if sel.any() else {})
    host = []
    for _ in range(iters):
        sm = TO.TemporalBEV()
        t0 = time.perf_counter()
        for f in parsed:
            if f:
                sm(f, 0)
        host.append((time.perf_counter() - t0) * 1e6 / T)
    return round(float(np.median(host)), 1)


def params():
    return dict(state_dict=synth.bev_damp_cam_offsets(synth.bev_state_dict(0)), smpla_pack=synth.smpl_pack(0, num_betas=11),
                smil_pack=synth.smpl_pack(1))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--precision", default="bf16", choices=["bf16", "tf32", "fp32"])
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--frames", type=int, default=256)
    ap.add_argument("--iters", type=int, default=3)
    a = ap.parse_args()
    v = Video(a.frames, a.batch)
    flags = ["--precision", a.precision, "--max_batch", str(a.batch)]
    torch.cuda.synchronize()
    m0 = torch.cuda.memory_allocated()
    plain = BEV(bev_settings(flags), **params())
    m1 = torch.cuda.memory_allocated()
    tm = BEV(bev_settings(flags + ["-t"]), **params())
    m2 = torch.cuda.memory_allocated()
    res = {}
    measure(v, plain, "plain", a.iters, res)
    measure(v, tm, "t", a.iters, res)
    res["oracle_cpu_us_per_frame"] = oracle_cpu_us_per_frame(v, plain, a.iters)
    name, power = card()
    counts = [len(c) for c in v.cells]
    res.update(people_per_frame=[min(counts), max(counts)], frames=v.T, batch=v.B, precision=a.precision,
               extra_device_mb=round(((m2 - m1) - (m1 - m0)) / 2**20, 1), gpu=name, power_limit=power, iters=a.iters)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
