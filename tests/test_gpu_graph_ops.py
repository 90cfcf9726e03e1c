"""Every op of the shipped conv graphs, checked in place against a float64 reference computed from its own inputs.

Graphs and batches (all with u8 frames):
  - ROMP bf16 (graph.build_romp) at batch 64, the benchmarked configuration; ROMP TF32 at batch 34; ROMP fp32 (the SIMT
    engine) at batch 5;
  - ROMP with the ResNet-50 backbone (graph.build_romp_resnet50, --backbone resnet50): bf16 at batch 64 (the CLI
    default), TF32 at batch 34, fp32 at batch 5;
  - BEV G1 and G2 (the bird's-eye Conv1d stack): bf16 at batches 34 and 136, TF32 at 34 and 16, fp32 at 5 and 16 (G2 runs
    on the SIMT engine outside bf16).
A persistent tensor-core kernel loops over tiles, so a scheduling bug can hide in the third tile a CTA runs (the fused block
kernel flips its mbarrier parity every tile).  The batches are picked so that the ops reach that tile where one graph fits
comfortably on the device; an op that needs more than 2 x 132 / tiles-per-frame frames for it (the unmerged 1x1 256->32
fuse conv of the last HRNet stage, 2 tiles per 16x16 frame on 132 CTAs) is run once more on its own, with its recorded
weights and its real input frames repeated, at a batch that gives some CTA 3 tiles (133).  The describe() plan of that
rerun must equal the graph's.  A fused Bottleneck cannot run alone: the graph batch itself must give it 3 tiles (layer1
of both backbones has 128 tiles per frame).  The fp32 graphs have no persistent kernels, so they run at a small batch.

How an op is checked:
  1. The builder's library calls (add_tensor, add_const_tensor, add_conv, add_sum, add_maxpool, set_lane, finalize) are
     recorded through a proxy of the loaded library while the builder runs.
  2. The recorded graph is replayed with one maxpool "keeper" per internal tensor appended before finalize, so the buffer
     planner recycles nothing and every op's input, residual, sum terms and output survive the run.  A fused block's
     intermediate gets no keeper (a second reader would undo the fusion); a fused Bottleneck's two do, and the kernel
     then also stores them, so each of its three describe() lines is checked as a conv of its own.  The keepers are known
     by their output tensors (the ResNet-50 graph has a maxpool of its own).  The keeper net's op lines must equal the
     production net's: same engines, plans, pixel-pair folds, block and Bottleneck fusions and grids.
  3. After one run, each op is recomputed in float64 with torch on the GPU from the tensors it read, and every element of
     its output slice must lie within
         bf16 out: 2^-8 |v| + g A,   fp32 out: 2^-23 |v| + g A,   g = 2^-24 (K + 3),
     with v the float64 result, A the same op on |X|, |W|, |b|, |res| and K the reduction length.  The operands are those
     the engine multiplies: bf16 weights as recorded, TF32-rounded activations and weights on the tc-tf32 engine, the
     stem engine's bf16(w * 2/255).  ConvTranspose2d(4, 2, 1) is referenced by F.conv_transpose2d with K = 4 cin (2 x 2
     taps per input channel reach each output); the ResNet-50 7x7 stem multiplies the raw u8 values (the recorded weights
     carry the normalisation) and adds its one-frame fp32 bias map to every frame.  A fused block's reference
     intermediate is bf16(relu(conv1 + b1)), zero outside the frame; where conv1's float64 value lies within g A1 of a
     bf16 rounding midpoint the kernel may round the other way, so conv(|W2|, one ulp + g A1) is added there.  A sum is
     bounded by 2^-8 |v| + 2^-24 (n + 1) sum|terms|, 1.1**z by carrying z's bound through the power.  A maxpool is exact:
     it must equal the float64 max_pool2d(3, 2, padding 1) with -inf padding bit for bit.
  Output slices are checked after the whole run: a later op that writes into an earlier op's slice fails the check.
Negative controls mutate the reference of a few ops (one dropped tap of a conv, block, transposed conv or 7x7 stem, one
dropped bias, a residual taken from the neighbouring channel pair, a maxpool window shifted by one pixel) and must be
rejected; test_bound_calibration_cpu runs the same bound on the CPU against an fp32 implementation with another
summation order.

Whole-graph checks compare bits: production net (buffer reuse) vs keeper net for every graph; in bf16 also each frame at
batch 64 vs batch 1 and inside a batch of 7; for HRNet bf16 CUDA graph vs eager launches, concurrency lanes vs one stream,
and more than 16 distinct (frames, output) bindings, which clears the CUDA-graph cache (for G2: changes of the bv_in
pointer and of the batch, on which the Conv1d tensor map is re-encoded); for ResNet-50 bf16 u8 frames vs fp32 frames
holding the same integers.

Measured on one H100 80GB HBM3 at a 700 W power limit (torch's peak allocation plus the keeper net's workspace; weights not counted), with the
runtime of each test including the whole-graph checks:
  ROMP bf16, batch 64: 12.0 GiB (9.8 GiB keeper workspace), 10-14 s;   ROMP TF32, batch 34: 15.4 GiB, 4 s;
  ROMP fp32, batch 5: 2.6 GiB, 2 s;
  ROMP ResNet-50 bf16, batch 64: 9.8 GiB (7.6 GiB keeper workspace), 7 s;   TF32, batch 34: 9.8 GiB, 4 s;
  ROMP ResNet-50 fp32, batch 5: 1.8 GiB, 2 s;
  BEV bf16 G1, batch 34: 7.8 GiB;  G2, batch 136: 1.2 GiB;  test 4.5-5.3 s;
  BEV TF32 G1, batch 34: 16.9 GiB;  G2, batch 16: 0.9 GiB;  test 5 s;   BEV fp32 G1, batch 5: 2.8 GiB;  G2: 0.3 GiB;  2 s.
"""
import ctypes as C
import math
import re
import time

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from romp_b200 import _lib, graph, synth
from romp_b200._lib import BF16, F32, U8, ConvDesc, SumDesc
from tests.gpu_util import TD, conv_ref, round_tf32

ROUND = {BF16: 2.0 ** -8, F32: 2.0 ** -23}
TAPS = {1: 1, 3: 9, 7: 49, 13: 3, 42: 16}
F32_11 = float(np.float32(1.1))          # powf(1.1f, x): the model's fp32 arithmetic
CHUNK = 1 << 24                          # float64 elements per reference chunk


# ---------------------------------------------------------------------------------------------------------------------
# reference and bound (pure torch: shared by the GPU checks and the CPU calibration test)
# ---------------------------------------------------------------------------------------------------------------------
def gamma(K):
    return 2.0 ** -24 * (K + 3)


def _nchw(t):
    return t.permute(0, 3, 1, 2)


def conv_linear(x, w, b, *, stride=1, up=1, transpose=False):
    """the convolution of a conv op, before its residual, ReLU and power: x NHWC, w, b float64 tensors, on x's device.
    w: OIHW, or [O, I, 3] (Conv1d along W, ksize code 13); transpose: ConvTranspose2d(4, 2, 1) with w in PyTorch's
    [cin, cout, 4, 4] layout (ksize code 42)"""
    if transpose:
        return F.conv_transpose2d(_nchw(x), w, b, stride=2, padding=1).permute(0, 2, 3, 1)
    return conv_ref(x, w, b, stride=stride, up=up, device=x.device, dtype=torch.float64)


def normalise_input(x):
    """input_norm of a conv op: raw 0..255 values -> x / 255 * 2 - 1 (model.py:385)"""
    return x / 255.0 * 2.0 - 1.0


def pow_f32_11(z):
    """the pow_channel of a conv op: powf(1.1f, z), the model's fp32 cam scale"""
    return torch.pow(torch.tensor(F32_11, dtype=torch.float64, device=z.device), z)


def conv_bound(x, w, b, *, stride=1, relu=False, res=None, up=1, pow_channel=-1, out_dt=BF16, input_norm=0, transpose=False):
    """float64 result v and per-element bound of one conv op; x, res: NHWC float64 (res may have one frame), w, b float64
    tensors.  input_norm: x holds raw 0..255 values; the kernel's normalised fp32 input carries 2^-22 absolute error.
    transpose: ConvTranspose2d(4, 2, 1) with w in PyTorch's [cin, cout, 4, 4] layout; each output sums 2 x 2 taps per
    input channel, so K = 4 cin."""
    if input_norm:
        x = normalise_input(x)
    if transpose:
        K = 4 * w.shape[0]
    else:
        K = w.shape[1] * (w.shape[2] * (w.shape[3] if w.ndim == 4 else 1))
    kw = dict(stride=stride, up=up, transpose=transpose)
    z = conv_linear(x, w, b, **kw)
    ax = x.abs() + (2.0 ** -22 if input_norm else 0.0)
    A = conv_linear(ax, w.abs(), None if b is None else b.abs(), **kw)
    if res is not None:
        z = z + res
        A = A + res.abs()
    if relu:
        z = z.clamp_min(0)
    v = z.clone()
    bound = ROUND[out_dt] * v.abs() + gamma(K) * A
    if pow_channel >= 0:
        zc = z[..., pow_channel]
        bz = gamma(K) * A[..., pow_channel] + 2.0 ** -23 * zc.abs()
        vc = pow_f32_11(zc)
        v[..., pow_channel] = vc
        bound[..., pow_channel] = vc * (F32_11 ** bz - 1) + 2.0 ** -21 * vc
    return v, bound


def _bf16_neighbours(m):
    """-> (bf16 rounding of m >= 0, distance of m to the nearest bf16 rounding midpoint, larger spacing around it)"""
    r = m.to(torch.bfloat16)
    bits = r.view(torch.int16).to(torch.int32)
    up = (bits + 1).to(torch.int16).view(torch.bfloat16).double()
    dn = (bits - 1).clamp_min(0).to(torch.int16).view(torch.bfloat16).double()
    rd = r.double()
    dist = torch.minimum((m - (rd + up) / 2).abs(), (m - (rd + dn) / 2).abs())
    return rd, dist, torch.maximum(up - rd, rd - dn)


def block_bound(x, w1, b1, w2, b2):
    """fused BasicBlock relu(conv2(bf16(relu(conv1(x) + b1))) + b2 + x): (v, bound); x NHWC float64"""
    K = w1.shape[1] * 9
    kw = dict(device=x.device, dtype=torch.float64)
    raw = conv_ref(x, w1, b1, **kw)
    A1 = conv_ref(x.abs(), w1.abs(), b1.abs(), **kw)
    mid, dist, spacing = _bf16_neighbours(raw.clamp_min(0))
    g1 = gamma(K) * A1
    # the kernel's fp32 conv1 may round to the other side of a midpoint (or of the ReLU) only within g1 of it
    dmid = torch.where((dist <= g1) & (raw >= -g1), spacing + g1, torch.zeros_like(g1))
    v = conv_ref(mid, w2, b2, res=x, relu=True, **kw)
    A2 = conv_ref(mid.abs(), w2.abs(), b2.abs(), res=x.abs(), **kw)
    bound = ROUND[BF16] * v.abs() + gamma(K) * A2 + conv_ref(dmid, w2.abs(), None, **kw)
    return v, bound


def sum_terms(base, terms, ups):
    """base + sum_k nearest_up(term_k, ups[k]); base, terms NHWC (already sliced)"""
    v = base.clone()
    for t, u in zip(terms, ups):
        if u > 1:
            t = t.repeat_interleave(u, 1).repeat_interleave(u, 2)
        v = v + t
    return v


def sum_bound(base, terms, ups, relu, out_dt):
    """fuse-layer sum act(base + sum_k nearest_up(term_k)); base, terms NHWC float64 (already sliced)"""
    v = sum_terms(base, terms, ups)
    a = sum_terms(base.abs(), [t.abs() for t in terms], ups)
    if relu:
        v = v.clamp_min(0)
    return v, ROUND[out_dt] * v.abs() + 2.0 ** -24 * (len(terms) + 1) * a


def maxpool_ref(x, shift=0):
    """MaxPool2d(3, 2, padding 1) of NHWC float64 x with -inf padding (a max is exact: no bound); shift moves every
    window `shift` pixels down and right"""
    xp = F.pad(_nchw(x), (1 - shift, 1 + shift, 1 - shift, 1 + shift), value=-math.inf)
    return F.max_pool2d(xp, 3, 2).permute(0, 2, 3, 1)


def excess(got, v, bound):
    """(worst |err| / bound, number of elements over the bound)"""
    err = (got.double() - v).abs()
    over = int((err > bound).sum())
    ratio = (err / bound.clamp_min(1e-300)).masked_fill(err == 0, 0.0)
    return float(ratio.max()), over


# ---------------------------------------------------------------------------------------------------------------------
# recording the builders' library calls
# ---------------------------------------------------------------------------------------------------------------------
class Recorder:
    """Proxy of the loaded library: forwards every call and records, per created net, the graph-building ones.
    finalize_batch: optional max_batch override per net index (in creation order)."""

    def __init__(self, lib, finalize_batch=None):
        self._lib = lib
        self.nets = []
        self.finalize_batch = finalize_batch or {}

    def __getattr__(self, name):
        return getattr(self._lib, name)

    def _rec(self, net):
        return next(r for r in self.nets if r["net"] == net)

    def b200romp_net_create(self, dev):
        net = self._lib.b200romp_net_create(dev)
        self.nets.append(dict(net=net, calls=[], tensors={}, max_batch=None))
        return net

    def b200romp_net_add_tensor(self, net, H, W, Cc, dt, nchw, ext):
        t = self._lib.b200romp_net_add_tensor(net, H, W, Cc, dt, nchw, ext)
        r = self._rec(net)
        r["calls"].append(("tensor", t, (H, W, Cc, dt, nchw, ext)))
        r["tensors"][t] = dict(H=H, W=W, C=Cc, dt=dt, nchw=nchw, ext=ext, const=False)
        return t

    def b200romp_net_add_const_tensor(self, net, H, W, Cc, dt, ptr):
        data = np.ctypeslib.as_array(C.cast(ptr, C.POINTER(C.c_float)), (H * W * Cc,)).copy()
        t = self._lib.b200romp_net_add_const_tensor(net, H, W, Cc, dt, ptr)
        r = self._rec(net)
        r["calls"].append(("const", t, (H, W, Cc, dt, data)))
        r["tensors"][t] = dict(H=H, W=W, C=Cc, dt=dt, nchw=0, ext=0, const=True)
        return t

    def b200romp_net_add_conv(self, net, dref, wp, bp):
        d = ConvDesc()
        C.memmove(C.byref(d), C.byref(dref._obj), C.sizeof(ConvDesc))
        w = np.ctypeslib.as_array(wp, (d.cout * d.cin * TAPS[d.ksize],)).copy()
        b = None if not bp else np.ctypeslib.as_array(bp, (d.cout,)).copy()
        op = self._lib.b200romp_net_add_conv(net, dref, wp, bp)
        self._rec(net)["calls"].append(("conv", op, (d, w, b)))
        return op

    def b200romp_net_add_sum(self, net, sref):
        s = SumDesc()
        C.memmove(C.byref(s), C.byref(sref._obj), C.sizeof(SumDesc))
        op = self._lib.b200romp_net_add_sum(net, sref)
        self._rec(net)["calls"].append(("sum", op, (s,)))
        return op

    def b200romp_net_add_maxpool(self, net, i, o):
        op = self._lib.b200romp_net_add_maxpool(net, i, o)
        self._rec(net)["calls"].append(("maxpool", op, (i, o)))
        return op

    def b200romp_net_set_lane(self, net, op, lane):
        self._rec(net)["calls"].append(("lane", None, (op, lane)))
        return self._lib.b200romp_net_set_lane(net, op, lane)

    def b200romp_net_finalize(self, net, max_batch):
        r = self._rec(net)
        r["max_batch"] = self.finalize_batch.get(self.nets.index(r), max_batch)
        return self._lib.b200romp_net_finalize(net, r["max_batch"])


def record(monkeypatch, build, finalize_batch=None):
    """run build() with the recording proxy installed; -> (build's result, [record per net])"""
    rec = Recorder(_lib.load(), finalize_batch)
    with monkeypatch.context() as m:
        m.setattr(_lib, "load", lambda: rec)
        out = build()
    return out, rec.nets


class Net:
    """a net made by replaying a record through the library, with optional keepers; or a builder's own net"""

    def __init__(self, lib, handle, tensors, max_batch):
        self.lib, self.net, self.tensors, self.max_batch = lib, handle, tensors, max_batch

    @classmethod
    def replay(cls, r, keep=(), max_batch=None):
        lib = _lib.load()
        net = lib.b200romp_net_create(0)
        assert net, lib.b200romp_last_error().decode()
        tensors = dict(r["tensors"])
        for kind, rid, args in r["calls"]:
            if kind == "tensor":
                got = lib.b200romp_net_add_tensor(net, *args)
            elif kind == "const":
                H, W, Cc, dt, data = args
                got = lib.b200romp_net_add_const_tensor(net, H, W, Cc, dt, data.ctypes.data_as(C.c_void_p))
            elif kind == "conv":
                d, w, b = args
                got = lib.b200romp_net_add_conv(net, C.byref(d), w.ctypes.data_as(C.POINTER(C.c_float)),
                                                None if b is None else b.ctypes.data_as(C.POINTER(C.c_float)))
            elif kind == "sum":
                got = lib.b200romp_net_add_sum(net, C.byref(args[0]))
            elif kind == "maxpool":
                got = lib.b200romp_net_add_maxpool(net, *args)
            else:
                _lib.check(lib.b200romp_net_set_lane(net, *args), "set_lane")
                continue
            assert got == rid, (kind, got, rid, lib.b200romp_last_error().decode())
        keepers = []
        for t in keep:
            # keepers: one maxpool reader per internal tensor.  Their outputs are external, so that no workspace buffer is
            # allocated after the first keeper: a kept tensor's buffer is freed after its keeper but never written again.
            s = tensors[t]
            k = _lib.check(lib.b200romp_net_add_tensor(net, (s["H"] - 1) // 2 + 1, (s["W"] - 1) // 2 + 1, s["C"], s["dt"], 0, 1))
            tensors[k] = dict(H=(s["H"] - 1) // 2 + 1, W=(s["W"] - 1) // 2 + 1, C=s["C"], dt=s["dt"], nchw=0, ext=1, const=False)
            _lib.check(lib.b200romp_net_add_maxpool(net, t, k), "keeper")
            keepers.append(k)
        mb = max_batch or r["max_batch"]
        _lib.check(lib.b200romp_net_finalize(net, mb), "finalize")
        n = cls(lib, net, tensors, mb)
        n.keepers = keepers
        return n

    def describe(self):
        buf = C.create_string_buffer(1 << 20)
        self.lib.b200romp_net_describe(self.net, buf, len(buf))
        return buf.value.decode()

    def op_lines(self):
        return [l for l in self.describe().splitlines() if l.startswith("op")]

    def alloc(self, t, batch):
        s = self.tensors[t]
        shape = (s["C"], s["H"], s["W"]) if s["nchw"] else (s["H"], s["W"], s["C"])
        return torch.empty((1 if s["const"] else batch,) + shape, dtype=TD[s["dt"]], device="cuda")

    def run(self, batch, binds, stream):
        for t, ten in binds.items():
            _lib.check(self.lib.b200romp_net_bind(self.net, t, C.c_void_p(ten.data_ptr())), "bind")
        _lib.check(self.lib.b200romp_net_run(self.net, batch, C.c_void_p(stream.cuda_stream)), "run")

    def read(self, t, batch, stream):
        out = self.alloc(t, batch)
        _lib.check(self.lib.b200romp_net_read_tensor(self.net, t, batch, C.c_void_p(out.data_ptr()), C.c_void_p(stream.cuda_stream)), "read")
        stream.synchronize()
        return out

    def destroy(self):
        if self.net:
            self.lib.b200romp_net_destroy(self.net)
            self.net = None




# ---------------------------------------------------------------------------------------------------------------------
# describe() lines -> ops
# ---------------------------------------------------------------------------------------------------------------------
TC_RE = re.compile(r"\[tc(-tf32)? k(\d) v(\d) nt(\d+) grid (\d+)x(\d+) smem \d+ stages \d+( pixel-pairs)?\]")
BLOCK_RE = re.compile(r"mid t(\d+).*\[tc-block grid (\d+) smem \d+( conv1 pixel-pairs conv2 pixel-pairs)?\]")
BOTTLENECK_RE = re.compile(r"\[tc-bottleneck conv(\d) of k1-k3-k1 grid (\d+) smem \d+\]")
IO_RE = re.compile(r" in t(\d+)\[.*? out t(\d+)\[")
OUT_RE = re.compile(r" out t(\d+)\[")


def ops_of(record, lines):
    """pair each op line of the production describe() with its recorded call(s); a fused Bottleneck prints one line per
    conv, each paired with that conv's call"""
    calls = [c for c in record["calls"] if c[0] in ("conv", "sum", "maxpool")]
    ops, i = [], 0
    for line in lines:
        if " block " in line:
            a, b = calls[i], calls[i + 1]
            assert a[0] == b[0] == "conv" and b[2][0].in_ == a[2][0].out
            m = BLOCK_RE.search(line)
            ops.append(dict(line=line, kind="block", convs=(a[2], b[2]), mid=int(m.group(1)), grid=int(m.group(2)),
                            fold=bool(m.group(3))))
            i += 2
            continue
        c = calls[i]
        i += 1
        if c[0] == "sum":
            ops.append(dict(line=line, kind="sum", sum=c[2][0]))
            continue
        io = IO_RE.search(line)
        io = (int(io.group(1)), int(io.group(2)))
        if c[0] == "maxpool":
            assert " maxpool " in line and io == c[2], line
            ops.append(dict(line=line, kind="maxpool", io=c[2]))
            continue
        assert c[0] == "conv", line
        d = c[2][0]
        assert io == (d.in_, d.out), line
        op = dict(line=line, kind="conv", conv=c[2], tc=None)
        m = TC_RE.search(line)
        if m:
            op["tc"] = dict(tf32=bool(m.group(1)), k=int(m.group(2)), v=int(m.group(3)), grid=int(m.group(5)),
                            fold=bool(m.group(7)), bracket=m.group(0))
        m = BOTTLENECK_RE.search(line)
        if m:
            op["tc"] = dict(bottleneck=int(m.group(1)), tf32=False, grid=int(m.group(2)), fold=False, bracket=m.group(0))
        ops.append(op)
    assert i == len(calls), "describe() has fewer op lines than the recorded graph"
    return ops


def op_class(op):
    if op["kind"] == "block":
        return "folded block" if op["fold"] else "block"
    if op["kind"] in ("sum", "maxpool"):
        return op["kind"]
    d, tc = op["conv"][0], op["tc"]
    if tc is None:       # the CUDA-core kernels: ConvTranspose2d(4, 2, 1), the 7x7 stem, the SIMT engine
        return {42: "deconv", 7: "k7"}.get(d.ksize, "SIMT")
    if "bottleneck" in tc:
        return "bottleneck"
    if tc["v"] == 3:
        return "conv1d" if d.ksize == 13 else "stem"
    if d.stride == 2:
        return "s2"
    return f"k{d.ksize}"


def tiles_per_cta(op, tensors, batch):
    """most tiles one CTA of a persistent tensor-core op runs at `batch` (None for other ops); -> (tiles, tiles per frame)"""
    if op["kind"] == "block":
        d = op["convs"][0][0]
        grid = op["grid"]
    elif op["kind"] == "conv" and op["tc"] is not None:
        d, grid = op["conv"][0], op["tc"]["grid"]
    else:
        return None, None
    t = tensors[d.out]
    Ho, Wo = t["H"] // d.upsample, t["W"] // d.upsample
    if d.ksize == 13:
        per_frame = Ho * (Wo // 128)
    else:
        per_frame = (Ho // 16) * ((Wo // 2 if (op.get("fold") or (op.get("tc") or {}).get("fold")) else Wo) // 8)
    n = per_frame * batch
    return -(-n // min(grid, n)), per_frame


# ---------------------------------------------------------------------------------------------------------------------
# checking one op
# ---------------------------------------------------------------------------------------------------------------------
def check_op(op, read, batch, frames=None, mutate=None):
    """-> (worst |err|/bound, elements over the bound, input nonzero fraction, output nonzero).  read(t) -> NHWC tensor of
    the whole batch (NCHW outputs already permuted); mutate(kind, arrays) edits the reference's operands in place."""
    sel = range(batch) if frames is None else frames
    worst, over, nz_in, nz_out = 0.0, 0, 0.0, False
    if op["kind"] == "sum":
        s = op["sum"]
        out_t = read(s.out)
        base = read(s.base)
        terms = [read(s.term[k])[..., s.term_c_off[k]:s.term_c_off[k] + out_t.shape[-1]] for k in range(s.n_terms)]
        ups = [s.up[k] for k in range(s.n_terms)]
        if mutate:
            mutate("sum", terms)
        nz_in = float((base != 0).float().mean())
        v, bnd = sum_bound(base.double(), [t.double() for t in terms], ups, bool(s.relu), _dt(out_t))
        r, o = excess(out_t, v, bnd)
        return r, o, nz_in, bool((out_t != 0).any())
    if op["kind"] == "maxpool":
        x_all, out_all = read(op["io"][0]), read(op["io"][1])
        shift = [0]
        if mutate:
            mutate("maxpool", shift)
        nz_in = float((x_all != 0).float().mean())
        step = max(1, CHUNK // (x_all[0].numel() * 2))
        idx = list(sel)
        for i in range(0, len(idx), step):
            fr = idx[i:i + step]
            v = maxpool_ref(x_all[fr].double(), shift[0]).to(out_all.dtype).double()   # exact: must equal bit for bit
            over += int((out_all[fr].double() != v).sum())
        return (math.inf if over else 0.0), over, nz_in, bool((out_all != 0).any())
    if op["kind"] == "block":
        (d1, w1, b1), (d2, w2, b2) = op["convs"]
        Cc = d1.cin
        w1 = torch.from_numpy(w1.reshape(Cc, Cc, 3, 3)).cuda().double()
        w2 = torch.from_numpy(w2.reshape(Cc, Cc, 3, 3)).cuda().double()
        b1, b2 = (torch.zeros(Cc, dtype=torch.float64, device="cuda") if b is None else torch.from_numpy(b).cuda().double()
                  for b in (b1, b2))
        x_all = read(d1.in_)[..., d1.in_c_off:d1.in_c_off + Cc]
        if mutate:
            mutate("block", [w1, b1, w2, b2], x_all.double().abs().mean((0, 1, 2)))
        y_all = read(d2.out)[..., d2.out_c_off:d2.out_c_off + Cc]
        nz_in = float((x_all != 0).float().mean())
        step = max(1, CHUNK // (x_all[0].numel() * 4))
        idx = list(sel)
        for i in range(0, len(idx), step):
            fr = idx[i:i + step]
            v, bnd = block_bound(x_all[fr].double(), w1, b1, w2, b2)
            r, o = excess(y_all[fr], v, bnd)
            worst, over = max(worst, r), over + o
        return worst, over, nz_in, bool((y_all != 0).any())
    d, w, b = op["conv"]
    tc = op["tc"]
    transpose = d.ksize == 42          # ConvTranspose2d(4, 2, 1): PyTorch's [cin, cout, 4, 4] weights
    shape = (d.cout, d.cin, 3) if d.ksize == 13 else (d.cin, d.cout, 4, 4) if transpose else (d.cout, d.cin, d.ksize, d.ksize)
    wt = torch.from_numpy(w.reshape(shape)).cuda()
    bt = None if b is None else torch.from_numpy(b).cuda().double()
    x_all = read(d.in_)
    u8_stem = x_all.dtype == torch.uint8 and tc is not None
    if u8_stem:      # the stem engine multiplies bf16(w * 2/255) with the exact (x - 127.5)
        wt = (wt * (2.0 / 255.0)).bfloat16().double() * (255.0 / 2.0)
    elif tc is not None and tc["tf32"]:
        wt = round_tf32(wt)
    wt = wt.double()
    x_all = x_all[..., d.in_c_off:d.in_c_off + d.cin]
    if mutate:
        mutate("deconv" if transpose else "conv", [wt, bt], x_all.double().abs().mean((0, 1, 2)))
    out_all = read(d.out)[..., d.out_c_off:d.out_c_off + d.cout]
    res_all = None if d.res < 0 else read(d.res)[..., d.res_c_off:d.res_c_off + d.cout]
    if res_all is not None and mutate:
        res_all = res_all.clone()
        mutate("res", [res_all])
    nz_in = float((x_all != 0).float().mean())
    step = max(1, CHUNK // (out_all[0].numel() * 4))
    idx = list(sel)
    for i in range(0, len(idx), step):
        fr = idx[i:i + step]
        x = x_all[fr]
        x = round_tf32(x).double() if (tc is not None and tc["tf32"]) else x.double()
        res = None
        if res_all is not None:
            res = res_all[:1].double() if d.res_broadcast else res_all[fr].double()
        v, bnd = conv_bound(x, wt, bt, stride=d.stride, relu=bool(d.relu), res=res, up=d.upsample, pow_channel=d.pow_channel,
                            out_dt=_dt(out_all), input_norm=d.input_norm, transpose=transpose)
        r, o = excess(out_all[fr], v, bnd)
        worst, over = max(worst, r), over + o
    return worst, over, nz_in, bool((out_all != 0).any())


def _dt(t):
    return BF16 if t.dtype == torch.bfloat16 else F32


class Reader:
    """read-back of a net's tensors after one run, cached for the op being checked (NCHW maps as NHWC views)"""

    def __init__(self, net, batch, stream, binds):
        self.net, self.batch, self.stream, self.binds, self.cache = net, batch, stream, binds, {}

    def __call__(self, t):
        if t not in self.cache:
            if t in self.binds:
                ten = self.binds[t][:self.batch]
            else:
                ten = self.net.read(t, self.batch, self.stream)
            self.cache[t] = ten.permute(0, 2, 3, 1) if self.net.tensors[t]["nchw"] else ten
        return self.cache[t]

    def keep_only(self, ts):
        self.cache = {k: v for k, v in self.cache.items() if k in ts}


# ---------------------------------------------------------------------------------------------------------------------
# one graph: keepers, per-op checks, coverage, reruns of ops that cannot reach a third tile per CTA at the graph batch
# ---------------------------------------------------------------------------------------------------------------------
def internal_tensors(r, mids):
    written = set()
    for kind, _, args in r["calls"]:
        if kind in ("conv", "sum"):
            written.add(args[0].out)
        elif kind == "maxpool":
            written.add(args[1])
    return [t for t, s in r["tensors"].items()
            if t in written and not s["ext"] and not s["const"] and not s["nchw"] and t not in mids]


def external_binds(r, batch, inputs):
    """torch buffers the test owns for every external tensor: inputs as given, outputs zero-filled"""
    binds = {}
    for t, s in r["tensors"].items():
        if not s["ext"]:
            continue
        if t in inputs:
            binds[t] = inputs[t]
        else:
            shape = (s["C"], s["H"], s["W"]) if s["nchw"] else (s["H"], s["W"], s["C"])
            binds[t] = torch.zeros((batch,) + shape, dtype=TD[s["dt"]], device="cuda")
    return binds


def keeper_net(r, prod_lines):
    mids = {int(m.group(1)) for l in prod_lines for m in [re.search(r"mid t(\d+)", l)] if m}
    keep = internal_tensors(r, mids)
    net = Net.replay(r, keep=keep)
    lines = net.op_lines()
    # the keepers are the ops replay appended: known by their output tensors (the graph may have maxpools of its own)
    kept_out = set(net.keepers)
    body = [l for l in lines if int(OUT_RE.search(l).group(1)) not in kept_out]
    assert len(lines) - len(body) == len(keep)
    assert all(int(OUT_RE.search(l).group(1)) in kept_out for l in lines[len(body):]), "a keeper is not last"
    assert body == prod_lines, "the keepers changed a kernel choice:\n" + "\n".join(
        f"{a}\n{b}" for a, b in zip(body, prod_lines) if a != b)
    return net


def rerun_alone(op, read, graph_batch, need=3):
    """an op whose tiles cannot give some CTA `need` tiles at the graph batch, run on its own: its input (and residual)
    frames repeated to a batch that does, through an exact identity copy into internal tensors, with the recorded weights.
    -> (batch, tiles per CTA, worst ratio, elements over the bound)"""
    d, w, b = op["conv"]
    per = tiles_per_cta(op, {d.out: dict(H=read.net.tensors[d.out]["H"], W=read.net.tensors[d.out]["W"])}, 1)[1]
    B = 2 * op["tc"]["grid"] // per + 1
    xin = read(d.in_)
    rep = [i % graph_batch for i in range(B)]
    lib = _lib.load()
    net = lib.b200romp_net_create(0)
    ti = read.net.tensors[d.in_]
    to = read.net.tensors[d.out]
    tensors, calls = {}, []

    def tensor(H, W, Cc, dt, nchw=0, ext=0):
        t = _lib.check(lib.b200romp_net_add_tensor(net, H, W, Cc, dt, nchw, ext))
        tensors[t] = dict(H=H, W=W, C=Cc, dt=dt, nchw=nchw, ext=ext, const=False)
        return t

    def copy(src, Cc, dt):
        dst = tensor(tensors[src]["H"], tensors[src]["W"], Cc, dt)
        eye = np.eye(Cc, dtype=np.float32).reshape(Cc, Cc, 1, 1)
        dd = ConvDesc(src, 0, dst, 0, -1, 0, 0, Cc, Cc, 1, 1, 0, 1, 0, -1, _lib.ENGINE_SIMT)
        _lib.check(lib.b200romp_net_add_conv(net, C.byref(dd), eye.ctypes.data_as(C.POINTER(C.c_float)), None), "copy")
        return dst

    src = tensor(ti["H"], ti["W"], ti["C"], ti["dt"], ext=1)
    x = copy(src, ti["C"], ti["dt"])
    binds = {src: xin[rep].contiguous()}
    res = -1
    if d.res >= 0:
        tr = read.net.tensors[d.res]
        rsrc = tensor(tr["H"], tr["W"], tr["C"], tr["dt"], ext=1)
        res = copy(rsrc, tr["C"], tr["dt"])
        rin = read(d.res)
        binds[rsrc] = (rin[[0] * B] if tr["const"] else rin[rep]).contiguous()
    out = tensor(to["H"], to["W"], to["C"], to["dt"], to["nchw"], ext=int(to["ext"]))
    dd = ConvDesc()
    C.memmove(C.byref(dd), C.byref(d), C.sizeof(ConvDesc))
    dd.in_, dd.out, dd.res = x, out, res
    _lib.check(lib.b200romp_net_add_conv(net, C.byref(dd), w.ctypes.data_as(C.POINTER(C.c_float)),
                                         None if b is None else b.ctypes.data_as(C.POINTER(C.c_float))), "op")
    _lib.check(lib.b200romp_net_finalize(net, B), "finalize")
    n = Net(lib, net, tensors, B)
    line = n.op_lines()[-1]
    assert op["tc"]["bracket"] in line, f"rerun plan differs:\n{line}\n{op['line']}"
    if to["ext"]:
        binds[out] = n.alloc(out, B).zero_()
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        n.run(B, binds, stream)
    stream.synchronize()
    rd = Reader(n, B, stream, binds)
    alone = dict(op, conv=(dd, w, b))
    tiles = tiles_per_cta(alone, tensors, B)[0]
    r, o, _, _ = check_op(alone, rd, B)
    n.destroy()
    return B, tiles, r, o


def verify_graph(name, r, prod_lines, batch, inputs, report):
    """keeper net of record r at `batch`; every op checked.  -> (keeper net, its external binds, ops, stream)"""
    t0 = time.time()
    torch.cuda.reset_peak_memory_stats()
    net = keeper_net(r, prod_lines)
    binds = external_binds(r, batch, inputs)
    # every keeper writes its (unused) output into one shared scratch buffer
    sizes = [net.alloc(k, 1).nbytes for k in net.keepers]
    scratch = torch.empty(max(sizes) * batch, dtype=torch.uint8, device="cuda")
    kbinds = {k: scratch for k in net.keepers}
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        net.run(batch, {**binds, **kbinds}, stream)
    stream.synchronize()
    del kbinds, scratch
    ops = ops_of(r, prod_lines)
    read = Reader(net, batch, stream, binds)
    stats, bad, few_tiles = {}, [], []
    for k, op in enumerate(ops):
        worst, over, nz_in, nz_out = check_op(op, read, batch)
        read.keep_only(())
        cls = op_class(op)
        st = stats.setdefault(cls, [0, 0.0])
        st[0] += 1
        st[1] = max(st[1], worst)
        if over or not nz_out or nz_in < 0.05:
            bad.append(f"{op['line']}\n    -> {over} elements over the bound (worst ratio {worst:.3g}), input nonzero "
                       f"{nz_in:.3f}, output nonzero {nz_out}")
        tiles, _ = tiles_per_cta(op, net.tensors, batch)
        if tiles is not None and tiles < 3:
            few_tiles.append(op)
    reruns = []
    for op in few_tiles:
        # a fused op cannot run alone: its graph batch must give it 3 tiles on some CTA
        assert op["kind"] == "conv" and op_class(op) != "bottleneck", \
            f"{name}: fused op below 3 tiles per CTA at batch {batch}:\n{op['line']}"
        B, tiles, worst, over = rerun_alone(op, read, batch)
        read.keep_only(())
        reruns.append((op_class(op), op["line"].split(" [")[0], B, tiles, worst))
        stats[op_class(op)][1] = max(stats[op_class(op)][1], worst)
        assert tiles >= 3
        if over:
            bad.append(f"{op['line']}\n    -> alone at batch {B}: {over} elements over the bound (worst ratio {worst:.3g})")
    dt = time.time() - t0
    ws = net.lib.b200romp_net_workspace_bytes(net.net)
    peak = torch.cuda.max_memory_allocated() + ws
    lines = [f"== {name}: batch {batch}, {len(ops)} ops verified in {dt:.1f} s, peak device memory {peak / 2**30:.2f} GiB "
             f"(keeper net workspace {ws / 2**30:.2f} GiB + torch {torch.cuda.max_memory_allocated() / 2**30:.2f} GiB)"]
    for cls, (n, worst) in sorted(stats.items()):
        lines.append(f"   {cls:13s} {n:4d} ops   worst |err|/bound {worst:.3f}")
    min_tiles = min((tiles_per_cta(op, net.tensors, batch)[0] for op in ops if tiles_per_cta(op, net.tensors, batch)[0]),
                    default=None)
    n_tc = sum(1 for op in ops if tiles_per_cta(op, net.tensors, batch)[0])
    lines.append(f"   {n_tc} persistent tensor-core ops; {n_tc - len(few_tiles)} reach >= 3 tiles on some CTA at batch {batch}"
                 f" (fewest: {min_tiles}), {len(reruns)} rerun alone:")
    for cls, line, B, tiles, worst in reruns:
        lines.append(f"     {cls:6s} {line.strip()}  -> batch {B}, {tiles} tiles on CTA 0, worst |err|/bound {worst:.3f}")
    report("\n".join(lines))
    assert len(ops) == len(prod_lines)
    assert not bad, f"{name}: {len(bad)} ops fail:\n" + "\n".join(bad[:20])
    return net, binds, ops, stream, read


# ---------------------------------------------------------------------------------------------------------------------
# negative controls: the comparison must reject a wrong reference
# ---------------------------------------------------------------------------------------------------------------------
def drop_tap(which=0):
    """zero the tap of one output channel of the weight array `which` (0 = conv1 of a block) that contributes most: largest
    |w| times the mean |input| of its channel.  Synthetic weights leave some channels dead after a ReLU, so with the mean
    |input| known the output channel is the one of largest mean pre-activation sum(w * mean|input|) + b, else channel 5."""
    def f(kind, a, act=None):
        if kind not in ("conv", "block", "deconv"):
            return
        i = 2 * which if kind == "block" else 0
        w, b = a[i], a[i + 1]
        if kind == "deconv":      # [cin, cout, 4, 4] -> a [cout, cin, 4, 4] view
            w = w.transpose(0, 1)
        co = 5
        score = w[co].abs()
        if act is not None and i == 0:
            act = act.reshape((-1,) + (1,) * (w.ndim - 2))
            pre = (w * act).flatten(1).sum(1) + (0 if b is None else b)
            co = int(pre.argmax())
            score = w[co].abs() * act
        taps = w[co]
        taps[torch.unravel_index(score.argmax(), score.shape)] = 0
    return f


def drop_bias():
    """zero the largest-magnitude bias of a conv"""
    def f(kind, a, act=None):
        if kind == "conv":
            a[1][a[1].abs().argmax()] = 0
    return f


def swap_res_pair(ch):
    def f(kind, a, act=None):
        if kind == "res":
            a[0][..., ch:ch + 2] = a[0][..., ch + 2:ch + 4].clone()
    return f


def shift_window():
    """every maxpool window of the reference one pixel down and right: it starts at 2 oy instead of 2 oy - 1"""
    def f(kind, a, act=None):
        if kind == "maxpool":
            a[0] = 1
    return f


def negative_controls(ops, read, batch, report):
    """each mutation of the reference must be rejected by the bound"""
    def first(pred):
        return next(op for op in ops if pred(op))

    tries = []
    for cls, what, mut in (("folded block", "folded 32-channel block, one tap", drop_tap()),
                           ("block", "64-channel block, one tap", drop_tap()),
                           ("k7", "7x7 stem, one tap", drop_tap()),
                           ("maxpool", "maxpool, window shifted by one pixel", shift_window())):
        if any(op_class(op) == cls for op in ops):
            tries.append((what, first(lambda o: op_class(o) == cls), mut))
    deconvs = [op for op in ops if op_class(op) == "deconv"]
    if deconvs:     # the shortest reduction: one of the 8192 taps of the 2048-channel one is within 2^-24 (K + 3) A
        tries.append(("transposed conv, one tap", min(deconvs, key=lambda o: o["conv"][0].cin), drop_tap()))
    # by descriptor, on any engine: a stride-2 1x1 or 3x3 conv of activations (not the u8 stem)
    tries.append(("stride-2 conv, one tap", first(lambda o: o["kind"] == "conv" and o["conv"][0].stride == 2 and
                                                  o["conv"][0].ksize in (1, 3) and
                                                  read.net.tensors[o["conv"][0].in_]["dt"] != U8), drop_tap()))
    heads = [op for op in ops if op["kind"] == "conv" and read.net.tensors[op["conv"][0].out]["nchw"]]
    if heads:
        tries.append(("head output conv, its largest bias", heads[-1], drop_bias()))
    tries.append(("residual of channels 2..3 from 4..5", first(lambda o: o["kind"] == "conv" and o["conv"][0].res >= 0
                                                               and o["conv"][0].cout >= 8 and not o["conv"][0].res_broadcast),
                  swap_res_pair(2)))
    frames = [0, batch - 1]
    for what, op, mut in tries:
        worst, over, _, _ = check_op(op, read, batch, frames=frames, mutate=mut)
        read.keep_only(())
        report(f"   negative control {what}: {over} elements over the bound (worst ratio {worst:.3g}) -> rejected")
        assert over > 0, f"negative control not rejected: {what} on\n{op['line']}"


# ---------------------------------------------------------------------------------------------------------------------
# fixtures and the graphs
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def romp_sd():
    return synth.romp_state_dict(0)


@pytest.fixture(scope="module")
def bev_sd():
    return synth.bev_state_dict(0)


@pytest.fixture(scope="module")
def resnet50_sd():
    return synth.resnet50_state_dict(0)


def _say(s):
    print(s, flush=True)


def _frames(B, seed):
    return torch.from_numpy(synth.synthetic_frames(B, seed=seed)).cuda()


def _outputs(net, io, keys, batch, frames, stream):
    binds = {io["frames"]: frames}
    outs = {}
    for k in keys:
        outs[k] = net.alloc(io[k], batch).zero_()
        binds[io[k]] = outs[k]
    with torch.cuda.stream(stream):
        net.run(batch, binds, stream)
    stream.synchronize()
    return outs


def _builder_net(nb, r):
    """a builder's own (production) net, with the tensor table of its record"""
    return Net(_lib.load(), nb.net, dict(r["tensors"]), r["max_batch"])


def _check_batch_invariance(prod, io, keys, frames, kept, stream):
    """frame i alone and inside a batch of 7 gives the bits of frame i of the full batch"""
    batch = frames.shape[0]
    for i in (0, batch // 2 - 1, batch - 1):
        one = _outputs(prod, io, keys, 1, frames[i:i + 1].contiguous(), stream)
        lo = min(max(i - 3, 0), batch - 7)
        seven = _outputs(prod, io, keys, 7, frames[lo:lo + 7].contiguous(), stream)
        for k in keys:
            assert torch.equal(one[k][0], kept[k][i]), f"{k}: frame {i} at batch 1 differs from batch {batch}"
            assert torch.equal(seven[k][i - lo], kept[k][i]), f"{k}: frame {i} in a batch of 7 differs"


@pytest.mark.gpu
@pytest.mark.parametrize("precision,batch", [("bf16", 64), ("tf32", 34), ("fp32", 5)])
def test_romp_graph_ops(monkeypatch, romp_sd, precision, batch):
    t0 = time.time()
    torch.cuda.synchronize()
    (nb, io), (r,) = record(monkeypatch, lambda: graph.build_romp(romp_sd, 0, precision, U8, batch))
    prod = _builder_net(nb, r)
    prod_lines = prod.op_lines()
    frames = _frames(batch, seed=21)
    net, binds, ops, stream, read = verify_graph(f"ROMP {precision}", r, prod_lines, batch, {io["frames"]: frames}, _say)
    negative_controls(ops, read, batch, _say)
    keys = ("center_maps", "params_maps")
    kept = {k: binds[io[k]] for k in keys}
    net.destroy()
    read.cache.clear()

    # buffer reuse: the production net computes the same bits as the net that keeps every tensor
    outs = _outputs(prod, io, keys, batch, frames, stream)
    for k in keys:
        assert torch.equal(outs[k], kept[k]), f"{k}: production net differs from the keeper net"
    if precision == "bf16":
        _check_batch_invariance(prod, io, keys, frames, kept, stream)
        # the CUDA-graph cache holds 16 bindings: 18 distinct (frames, output) buffers make it clear itself
        alive = []                       # every binding stays allocated: no address repeats
        for j in range(18):
            alive.append(frames[j:j + 2].clone())
            got = _outputs(prod, io, keys, 2, alive[-1], stream)
            alive.append(got)
            for k in keys:
                assert torch.equal(got[k], kept[k][j:j + 2]), f"{k}: binding {j} after the graph cache cycled"
        # eager launches and concurrency lanes compute the same bits as the CUDA graph of one stream
        for env in ("B200ROMP_NO_GRAPH", "B200ROMP_LANES"):
            with monkeypatch.context() as m:
                m.setenv(env, "1")
                nb2, _ = graph.build_romp(romp_sd, 0, precision, U8, 8)
            other = _builder_net(nb2, r)
            got = _outputs(other, io, keys, 8, frames[:8].contiguous(), stream)
            other.destroy()
            for k in keys:
                assert torch.equal(got[k], kept[k][:8]), f"{k}: {env}=1 differs"
    prod.destroy()
    _say(f"   ROMP {precision}: total {time.time() - t0:.1f} s")


@pytest.mark.gpu
@pytest.mark.parametrize("precision,batch", [("bf16", 64), ("tf32", 34), ("fp32", 5)])
def test_romp_resnet50_graph_ops(monkeypatch, resnet50_sd, precision, batch):
    """ROMP with the ResNet-50 backbone (--backbone resnet50): the 7x7 stem on raw u8 frames, MaxPool2d(3, 2, 1), the
    1x1 convs to 512 / 1024 channels, the fused Bottlenecks of layer1 (bf16), the K-split 256-channel stride-2 conv of
    layer3.0, the SIMT convs of 512..2048 input channels and the three ConvTranspose2d(4, 2, 1)."""
    t0 = time.time()
    torch.cuda.synchronize()
    (nb, io), (r,) = record(monkeypatch, lambda: graph.build_romp_resnet50(resnet50_sd, 0, precision, U8, batch))
    prod = _builder_net(nb, r)
    frames = _frames(batch, seed=51)
    name = f"ROMP ResNet-50 {precision}"
    net, binds, ops, stream, read = verify_graph(name, r, prod.op_lines(), batch, {io["frames"]: frames}, _say)
    classes = {op_class(op) for op in ops}
    assert {"k7", "maxpool", "deconv", "SIMT"} <= classes, classes
    assert precision != "bf16" or "bottleneck" in classes, classes
    negative_controls(ops, read, batch, _say)
    keys = ("center_maps", "params_maps")
    kept = {k: binds[io[k]] for k in keys}
    net.destroy()
    read.cache.clear()

    outs = _outputs(prod, io, keys, batch, frames, stream)
    for k in keys:
        assert torch.equal(outs[k], kept[k]), f"{k}: production net differs from the keeper net"
    if precision == "bf16":
        _check_batch_invariance(prod, io, keys, frames, kept, stream)
        # the stem multiplies raw values: fp32 frames holding the same integers give the same bits as u8 frames
        nbf, iof = graph.build_romp_resnet50(resnet50_sd, 0, precision, F32, 8)
        other = _builder_net(nbf, r)
        got = _outputs(other, iof, keys, 8, frames[:8].float(), stream)
        other.destroy()
        for k in keys:
            assert torch.equal(got[k], kept[k][:8]), f"{k}: fp32 frames differ from u8 frames"
    prod.destroy()
    _say(f"   {name}: total {time.time() - t0:.1f} s")


# G1 at batch 34 takes every tensor-core op but one (see the module docstring) to 3 tiles per CTA, in bf16 and TF32 alike;
# the fp32 graphs are SIMT only, and G2 outside bf16 is too.
BEV_BATCHES = {"bf16": (34, 136), "tf32": (34, 16), "fp32": (5, 16)}


def _bev_graph_ops(monkeypatch, bev_sd, precision):
    """BEV's G1 and G2 at `precision`: every op checked, negative controls on G1, production vs keeper net, G2 bindings"""
    t0 = time.time()
    b1, b2 = BEV_BATCHES[precision]
    (g1, io1, g2, io2), (r1, r2) = record(monkeypatch, lambda: graph.build_bev(bev_sd, 0, precision, U8, b1),
                                         finalize_batch={1: b2})
    p1, p2 = _builder_net(g1, r1), _builder_net(g2, r2)
    frames = _frames(b1, seed=33)
    keys1 = ("maps_fv", "fv_feats", "img_feats")
    net1, binds1, ops1, stream, read1 = verify_graph(f"BEV {precision} G1", r1, p1.op_lines(), b1,
                                                     {io1["frames"]: frames}, _say)
    negative_controls(ops1, read1, b1, _say)
    kept1 = {k: binds1[io1[k]] for k in keys1}
    net1.destroy()
    read1.cache.clear()
    outs = _outputs(p1, io1, keys1, b1, frames, stream)
    for k in keys1:
        assert torch.equal(outs[k], kept1[k]), f"{k}: production G1 differs from the keeper net"
    p1.destroy()

    # G2 on a non-negative bird's-eye input (it is assembled from ReLU features)
    g = torch.Generator(device="cuda").manual_seed(7)
    bv = torch.randn(b2, 1, 128, 2560, generator=g, device="cuda").abs().to(TD[r2["tensors"][io2["bv_in"]]["dt"]])
    net2, binds2, ops2, stream, read2 = verify_graph(f"BEV {precision} G2", r2, p2.op_lines(), b2, {io2["bv_in"]: bv}, _say)
    kept2 = binds2[io2["bv_out"]]
    net2.destroy()
    read2.cache.clear()

    def g2_run(x, batch):
        out = p2.alloc(io2["bv_out"], batch).zero_()
        with torch.cuda.stream(stream):
            p2.run(batch, {io2["bv_in"]: x, io2["bv_out"]: out}, stream)
        stream.synchronize()
        return out

    assert torch.equal(g2_run(bv, b2), kept2), "bv_out: production G2 differs from the keeper net"
    # the Conv1d tensor map is re-encoded when bv_in moves or the batch changes: 18 bindings of varying batch
    alive = []
    for j in range(18):
        n = 1 + (j * 5) % 9
        lo = (j * 7) % (b2 - n)
        alive.append(bv[lo:lo + n].clone())
        alive.append(g2_run(alive[-1], n))
        assert torch.equal(alive[-1], kept2[lo:lo + n]), f"bv_out: binding {j} (batch {n})"
    p2.destroy()
    _say(f"   BEV {precision}: total {time.time() - t0:.1f} s")


@pytest.mark.gpu
def test_bev_graph_ops(monkeypatch, bev_sd):
    _bev_graph_ops(monkeypatch, bev_sd, "bf16")


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["tf32", "fp32"])
def test_bev_graph_ops_fp32_tensors(monkeypatch, bev_sd, precision):
    """BEV with fp32 activations: G1 on the TF32 engine (16 image-feature channels on the SIMT engine) or the SIMT
    engine, G2 on the SIMT engine"""
    _bev_graph_ops(monkeypatch, bev_sd, precision)


# ---------------------------------------------------------------------------------------------------------------------
# the bound itself, on the CPU
# ---------------------------------------------------------------------------------------------------------------------
def _alt_conv(x, w, b, stride, res, relu, parts=4, transpose=False):
    """another implementation: fp32 torch on the CPU, K split into channel groups summed in reverse order, bf16 output.
    transpose: ConvTranspose2d(4, 2, 1) with w [cin, cout, 4, 4]; a one-frame residual is broadcast over the batch."""
    cin = w.shape[0 if transpose else 1]
    step = max(1, cin // parts)
    acc = None
    for c0 in reversed(range(0, cin, step)):
        xs = _nchw(x[..., c0:c0 + step]).float()
        if transpose:
            y = F.conv_transpose2d(xs, w[c0:c0 + step].float(), None, stride=2, padding=1)
        else:
            y = F.conv2d(xs, w[:, c0:c0 + step].float(), None, stride=stride, padding=w.shape[-1] // 2)
        acc = y if acc is None else acc + y
    acc = acc + b.float()[None, :, None, None]
    if res is not None:
        acc = acc + _nchw(res).float()
    if relu:
        acc = acc.clamp_min(0)
    return acc.permute(0, 2, 3, 1).bfloat16()


@pytest.mark.parametrize("k,cin,cout,stride,hw,res", [(3, 64, 64, 1, 16, True), (3, 32, 32, 1, 32, True), (1, 256, 32, 1, 8, False),
                                                       (3, 32, 64, 2, 32, False), (1, 64, 256, 1, 16, True),
                                                       (42, 64, 32, 2, 8, False), (7, 3, 64, 2, 32, "broadcast")])
def test_bound_calibration_cpu(k, cin, cout, stride, hw, res):
    """The per-element bound accepts a legitimate other implementation of the same op and rejects the mutations the GPU
    negative controls use: a dropped tap, a dropped bias, a residual from the neighbouring channel pair.
    k = 42 is ConvTranspose2d(4, 2, 1) (weights [cin, cout, 4, 4]); the 7x7 case is the ResNet-50 stem: raw u8 values
    times weights scaled by 1 / (255 std), plus a one-frame fp32 residual broadcast over the batch."""
    g = torch.Generator().manual_seed(k * 100 + cin + cout)
    transpose = k == 42
    if k == 7:
        x = torch.randint(0, 256, (3, hw, hw, cin), generator=g, dtype=torch.uint8)
        w = (torch.randn(cout, cin, k, k, generator=g) / math.sqrt(cin * k * k) / 57.0).bfloat16().double()
    elif transpose:
        x = torch.randn(3, hw, hw, cin, generator=g).clamp_min(0).bfloat16()
        w = (torch.randn(cin, cout, 4, 4, generator=g) / math.sqrt(4 * cin)).double()
    else:
        x = torch.randn(3, hw, hw, cin, generator=g).clamp_min(0).bfloat16()
        w = (torch.randn(cout, cin, k, k, generator=g) / math.sqrt(cin * k * k)).bfloat16().double()
    b = 0.1 * torch.randn(cout, generator=g, dtype=torch.float64)
    ho = 2 * hw if transpose else hw // stride
    if res == "broadcast":
        r = torch.randn(1, ho, ho, cout, generator=g)
    else:
        r = torch.randn(3, ho, ho, cout, generator=g).bfloat16() if res else None
    got = _alt_conv(x, w, b, stride, r, relu=True, transpose=transpose)
    rd = None if r is None else r.double()
    kw = dict(stride=stride, relu=True, transpose=transpose)
    v, bnd = conv_bound(x.double(), w, b, res=rd, **kw)
    worst, over = excess(got, v, bnd)
    print(f"k{k} s{stride} {cin}->{cout}: fp32 CPU implementation worst |err|/bound {worst:.3f}")
    assert over == 0 and worst < 1

    w2 = w.clone()
    flat = w2[5].reshape(-1)
    flat[flat.abs().argmax()] = 0
    assert excess(got, *conv_bound(x.double(), w2, b, res=rd, **kw))[1] > 0, "dropped tap accepted"
    b2 = b.clone()
    b2[b.abs().argmax()] = 0
    assert excess(got, *conv_bound(x.double(), w, b2, res=rd, **kw))[1] > 0, "dropped bias accepted"
    if res:
        r2 = rd.clone()
        r2[..., 2:4] = rd[..., 4:6]
        assert excess(got, *conv_bound(x.double(), w, b, res=r2, **kw))[1] > 0, "swapped residual accepted"


@pytest.mark.parametrize("cin", [32, 64])
def test_block_bound_calibration_cpu(cin):
    """The fused-block bound (bf16 intermediate with the midpoint allowance) accepts an fp32 CPU implementation that rounds
    its own intermediate to bf16, and rejects one dropped tap of conv1 or conv2."""
    g = torch.Generator().manual_seed(cin)
    x = torch.randn(2, 16, 24, cin, generator=g).clamp_min(0).bfloat16()
    w1 = (torch.randn(cin, cin, 3, 3, generator=g) / math.sqrt(9 * cin)).bfloat16().double()
    w2 = (torch.randn(cin, cin, 3, 3, generator=g) / math.sqrt(9 * cin)).bfloat16().double()
    b1 = 0.1 * torch.randn(cin, generator=g, dtype=torch.float64)
    b2 = 0.1 * torch.randn(cin, generator=g, dtype=torch.float64)
    mid = _alt_conv(x, w1, b1, 1, None, relu=True)
    got = _alt_conv(mid, w2, b2, 1, x, relu=True, parts=2)
    worst, over = excess(got, *block_bound(x.double(), w1, b1, w2, b2))
    print(f"block {cin}: fp32 CPU implementation worst |err|/bound {worst:.3f}")
    assert over == 0
    for which in (0, 1):
        ws = [w1.clone(), b1, w2.clone(), b2]
        drop_tap(which)("block", ws)
        assert excess(got, *block_bound(x.double(), *ws))[1] > 0, f"dropped tap of conv{which + 1} accepted"
