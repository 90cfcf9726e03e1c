"""Per-op device-time table of the ROMP conv net (b200romp_net_profile): which layers the step is spent in.

    python tools/op_profile.py [--batch 64] [--iters 5] > op_profile.md

Ops are launched one by one (no CUDA graph) with a CUDA event between them, so the numbers are warm-cache device
times in network order; FLOP counts are algorithmic (2*MAC of the conv at its own resolution).  Bytes are algorithmic too:
the input channel slice, the output and the residual read once each, at the activation size of the precision (2 bytes in
bf16, 4 otherwise; the few fp32 tensors of a bf16 net are counted at 2).  Low-intensity layers are bounded by these bytes,
not by FLOPs, so GB/s is the rate to set against the HBM bandwidth.  A fused BasicBlock op (`block k3`, conv_block_tc.cu)
counts the FLOPs of both convs and moves its input once and its output once: the intermediate stays in shared memory and
the residual is the block's own input, read from the staged input tile, so neither adds bytes.  A fused Bottleneck op
(conv_bottleneck_tc.cu, one describe() line per conv under one op number, shown here as `bottleneck k1-k3-k1`) counts the algorithmic FLOPs of its three convs (not conv1's recompute on
the tile halo) and moves its input once and its output once: both intermediates stay in shared memory and the residual,
its own input, is read again from L2."""
import argparse
import os
import re
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--top", type=int, default=400)
    ap.add_argument("--precision", type=str, default="bf16", choices=["bf16", "tf32", "fp32"])
    args = ap.parse_args()
    from romp_b200 import graph, synth, _lib

    torch.cuda.set_device(0)
    B = args.batch
    nb, io = graph.build_romp(synth.romp_state_dict(0), 0, args.precision, _lib.U8, max_batch=B)
    lib = nb.lib
    eb = 2 if args.precision == "bf16" else 4
    frames = torch.randint(0, 256, (B, 512, 512, 3), dtype=torch.uint8, device="cuda")
    ext = {}
    if io is not None:
        ext["frames"] = frames
        ext["center_maps"] = torch.empty(B, 1, 64, 64, device="cuda")
        ext["params_maps"] = torch.empty(B, 145, 64, 64, device="cuda")
        for k, t in ext.items():
            _lib.check(lib.b200romp_net_bind(nb.net, io[k], t.data_ptr()))
    us = nb.profile(B, args.iters)
    lines = []
    for l in nb.describe().splitlines():
        if not l.startswith("op"):
            continue
        m = re.search(r"k\d s1 +(\d+)->(\d+) +in (t\d+\[\S+).*\[tc-bottleneck conv(\d)", l)
        if m and m.group(4) != "1":   # conv2 / conv3 of the fused Bottleneck begun on the previous line: one op, one time
            lines[-1] = lines[-1].replace("->?", f"->{m.group(2)}" + ("->?" if m.group(4) == "2" else ""))
            continue
        if m:
            l = f"{l[:5]} wgmma   bottleneck k1-k3-k1 {m.group(1)}->{m.group(2)}->? in {m.group(3)}"
        lines.append(l)
    rows = []
    for l, t in zip(lines, us):
        if " sum " in l:
            rows.append((t, 0.0, 0.0, l))
            continue
        mb = re.search(r"block k3 s1 (\d+)->(\d+)->(\d+) in t\d+\[(\d+)x(\d+)x\d+\]", l)
        if mb:
            c0, c1, c2, H, W = (int(x) for x in mb.groups())
            rows.append((t, 2.0 * B * H * W * 9 * (c0 * c1 + c1 * c2), eb * B * H * W * (c0 + c2), l))
            continue
        mb = re.search(r"bottleneck k1-k3-k1 (\d+)->(\d+)->(\d+)->(\d+) in t\d+\[(\d+)x(\d+)x\d+\]", l)
        if mb:
            c0, c1, c2, c3, H, W = (int(x) for x in mb.groups())
            rows.append((t, 2.0 * B * H * W * (c0 * c1 + 9 * c1 * c2 + c2 * c3), eb * B * H * W * (c0 + c3), l))
            continue
        m = re.search(r"k(\d+) s(\d) +(\d+)->(\d+) +in t\d+\[(\d+)x(\d+)x\d+\]", l)
        k, s, cin, cout, H, W = (int(x) for x in m.groups())
        k2 = 3 if k == 13 else k * k
        ho, wo = H // s, W // s
        up = int(re.search(r"up(\d)", l).group(1))
        flop = 2.0 * B * ho * wo * cin * cout * k2
        nbytes = eb * B * (H * W * cin + ho * wo * up * up * cout * (2 if "res t-1" not in l else 1))
        rows.append((t, flop, nbytes, l))
    total = sum(r[0] for r in rows)
    tf = sum(r[1] for r in rows)
    tb = sum(r[2] for r in rows)
    print(f"# per-op profile, batch {B}: {len(rows)} ops, {total / 1000:.3f} ms, {tf / total / 1e6:.1f} TFLOP/s, {tb / total / 1e3:.0f} GB/s overall\n")
    # by class
    cls = {}
    for t, f, nb_, l in rows:
        if " sum " in l:
            ms = re.search(r"out t\d+\[(\d+)x\d+x(\d+)\]", l)
            a = cls.setdefault(f"sum @{ms.group(1)} c{ms.group(2)} terms{l.count('up')}", [0, 0.0, 0.0, 0.0])
            a[0] += 1; a[1] += t
            continue
        mb = re.search(r"(block k3|bottleneck k1-k3-k1) (?:s1 )?(\d+->\d+->\d+(?:->\d+)?) in t\d+\[(\d+)x", l)
        if mb:
            a = cls.setdefault(f"wgmma {mb.group(1)} {mb.group(2)} @{mb.group(3)} res", [0, 0.0, 0.0, 0.0])
            a[0] += 1; a[1] += t; a[2] += f; a[3] += nb_
            continue
        m = re.search(r"(wgmma|simt) +k(\d+) s(\d) +(\d+)->(\d+) +in t\d+\[(\d+)x", l)
        key = f"{m.group(1)} k{m.group(2)} s{m.group(3)} {m.group(4)}->{m.group(5)} @{m.group(6)}" + (" epi" + l.split("epi")[1][0] if "epi" in l else "") + \
              (" up" + re.search(r"up(\d)", l).group(1)) + (" res" if "res t-1" not in l else "")
        a = cls.setdefault(key, [0, 0.0, 0.0, 0.0])
        a[0] += 1; a[1] += t; a[2] += f; a[3] += nb_
    print("| class | ops | total us | share | avg us | TFLOP/s | GB/s |\n|---|---:|---:|---:|---:|---:|---:|")
    for k, (n, t, f, nb_) in sorted(cls.items(), key=lambda kv: -kv[1][1]):
        print(f"| {k} | {n} | {t:.1f} | {100 * t / total:.1f}% | {t / n:.1f} | {f / t / 1e6:.0f} | {nb_ / t / 1e3:.0f} |")
    print("\n| us | TFLOP/s | GB/s | op |\n|---:|---:|---:|---|")
    for t, f, nb_, l in sorted(rows, key=lambda r: -r[0])[:args.top]:
        print(f"| {t:.1f} | {f / t / 1e6:.0f} | {nb_ / t / 1e3:.0f} | `{l.strip()}` |")


if __name__ == "__main__":
    main()
