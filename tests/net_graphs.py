"""Seeded random conv graphs for libb200romp, built as the NetBuilder calls a graph builder would make.

generate(seed) returns a record in the format of test_gpu_graph_ops.Recorder (calls, tensors, max_batch), so that
test_gpu_graph_ops.Net.replay and verify_graph take it like a builder's graph.  Every graph is small (frames of 16-64
pixels, plus a 128x128 u8 frame for the stem and 16x128 maps for the Conv1d engine) and mixes

  - random ops over the tensors written so far: convs (ksize 1, 3, 7, 13 = Conv1d 1x3, 42 = ConvTranspose2d(4, 2, 1);
    stride 1 and 2; upsample; ReLU; residuals in bf16 or fp32, from a channel slice or broadcast from a const tensor;
    AUTO, WGMMA, TF32 and SIMT engines), sums of 1-4 terms (up 1-8, term_c_off) and maxpools, on lanes 0-3;
  - planted ops: items() below, a fixed share of them per seed, so that over SEEDS every kernel-selection branch of the
    library is reached: every reachable B2R_CASE row of conv_tc.cu in its direct-NHWC and its generic epilogue, the
    SWAP (kind 31), streamed (34), stem (33) and Conv1d (13) plans, every SIMT instantiation, the fused BasicBlock
    (folded and not), the fused Bottleneck (with and without stored intermediates), the fuse-sum kernels, maxpool, and
    near misses that must not fuse or must fall back to the SIMT engine.  Each planted op carries the plan it must get
    (expect), which the GPU test reads back from describe().

Rules every graph keeps (check_record restates them, test_net_graphs_cpu runs it over every seed):
  - the validity checks of add_conv (validate_desc), add_sum and add_maxpool in net.cu;
  - every channel an op reads of an internal tensor has been written by an earlier op, and each channel is written once
    (so the per-op check after the whole run sees every op's inputs and outputs as they were);
  - the aliasing rule of include/b200romp.h: a slice an op reads of its own output tensor is disjoint from the output
    slice (the identical-slice forms rewrite a tensor and are tested on their own);
  - NCHW tensors are external outputs; internal tensors are NHWC.

plan_workspace restates the buffer planner of b200romp_net_finalize on the op list as describe() reports it (after
fusion): linear-order liveness and exact-size free lists of 1 KiB-rounded frame_bytes * max_batch.
"""
import ctypes as C
import math
import re

import numpy as np

from romp_b200._lib import BF16, ENGINE_AUTO, ENGINE_SIMT, ENGINE_TF32, ENGINE_WGMMA, F32, U8, ConvDesc, SumDesc

SEEDS = range(160)
BATCH = 20                 # graph batch: the planted fused ops (64x64 frames) reach 3 tiles on some CTA of 132
DSIZE = {F32: 4, BF16: 2, U8: 1}
TAPS = {1: 1, 3: 9, 7: 49, 13: 3, 42: 16}


def out_hw(k, s, H, W):
    """net.cu conv_out_hw"""
    if k == 42:
        return 2 * H, 2 * W
    kh, kw = (1, 3) if k == 13 else (k, k)
    return (H + 2 * (kh // 2) - kh) // s + 1, (W + 2 * (kw // 2) - kw) // s + 1


def bf16_round(a):
    """round-to-nearest-even to bf16, kept as float32"""
    u = np.ascontiguousarray(a, dtype=np.float32).view(np.uint32).astype(np.uint64)
    u = ((u + 0x7FFF + ((u >> 16) & 1)) >> 16) << 16
    return u.astype(np.uint32).view(np.float32)


# ---------------------------------------------------------------------------------------------------------------------
# the TC dispatch table (conv_tc.cu B2R_CASE rows) and the rows no shape selects
# ---------------------------------------------------------------------------------------------------------------------
def b2r_rows(src):
    """(mode, cin, nt, eb) of every B2R_CASE row in the text of conv_tc.cu; mode 1 = 1x1, 3 = 3x3 s1, 2 = 3x3 s2"""
    return [tuple(int(x) for x in m) for m in re.findall(r"B2R_CASE\((\d), (\d+), (\d+), (\d)\)", src)]


def tc_nt(mode, cin, cout, eb):
    """conv_tc.cu tc_tile: the N tile of a plain (not streamed) plan, or None when the weights do not fit"""
    k = 1 if mode == 1 else 3
    if mode == 2:
        rowb = 64 if cin * eb >= 512 else (cin * eb if cin * eb < 128 else 128)
    else:
        rowb = 64 if (k == 3 and cin >= 128) else (cin * eb if cin * eb < 128 else 128)
    kch = cin // (rowb // eb)
    budget = 227 * 1024 - 2048
    bb = lambda n: k * k * kch * n * rowb
    nt = 64 if cout % 64 == 0 else 32
    if mode == 2:
        sub = lambda i: ((17 if i < 2 else 16) * (8 if i & 1 else 9) * rowb + 1023) // 1024 * 1024
        stage = sum(sub(i) for i in range(4))
        if nt == 64 and bb(64) + 2 * stage > budget and bb(32) + 2 * stage <= budget:
            nt = 32
        if nt == 64 and bb(64) + stage > budget:
            nt = 32
        return nt if bb(nt) + stage <= budget else None
    stage = ((16 + 2 * (k // 2)) * (8 + 2 * (k // 2)) * rowb + 1023) // 1024 * 1024
    if bb(nt) + 3 * stage > budget and nt == 64:
        nt = 32
    if bb(nt) + 2 * stage > budget and nt == 32:
        nt = 16
    return nt if bb(nt) + 2 * stage <= budget else None


def unreachable_rows(rows):
    """rows that no cout selects: a plain plan at that N tile needs more shared memory than there is, and the streamed
    plan (kind 34) takes the bf16 3x3 256-channel convs it could otherwise serve"""
    reach = set()
    for mode, cin, _, eb in rows:
        for cout in (32, 64, 96, 128, 192, 256):
            nt = tc_nt(mode, cin, cout, eb)
            if nt:
                reach.add((mode, cin, nt, eb))
    return [r for r in rows if r not in reach]


# ---------------------------------------------------------------------------------------------------------------------
# the generator
# ---------------------------------------------------------------------------------------------------------------------
class Graph:
    def __init__(self, seed, batch=BATCH):
        self.seed = seed
        self.rng = np.random.default_rng(seed)
        self.calls, self.tensors, self.written = [], {}, {}
        self.n_ops = 0
        self.lanes = {}
        self.inputs = []           # external tensors the caller fills
        self.expect = []           # (item, op ids, expected plan)
        self.pool = []             # internal NHWC tensors written whole
        self.ext_in = {}           # (H, W, dt) -> external input tensor
        self.batch = batch

    # ---- NetBuilder calls ------------------------------------------------------------------------------------------
    def tensor(self, H, W, Cc, dt, nchw=0, ext=0):
        t = len(self.tensors)
        self.calls.append(("tensor", t, (H, W, Cc, dt, nchw, ext)))
        self.tensors[t] = dict(H=H, W=W, C=Cc, dt=dt, nchw=nchw, ext=ext, const=False)
        self.written[t] = np.zeros(Cc, bool)
        return t

    def const(self, H, W, Cc):
        t = len(self.tensors)
        data = (0.5 * self.rng.standard_normal(H * W * Cc)).astype(np.float32)
        self.calls.append(("const", t, (H, W, Cc, F32, data)))
        self.tensors[t] = dict(H=H, W=W, C=Cc, dt=F32, nchw=0, ext=0, const=True)
        self.written[t] = np.ones(Cc, bool)
        return t

    def conv(self, i, o, cin, cout, k=3, s=1, in_off=0, out_off=0, res=-1, res_off=0, bcast=0, relu=1, up=1, norm=0,
             pw=-1, engine=ENGINE_AUTO, lane=0):
        assert self.written[i][in_off:in_off + cin].all(), "conv reads an unwritten channel"
        assert res < 0 or self.written[res][res_off:res_off + cout].all(), "conv adds an unwritten channel"
        assert not self.written[o][out_off:out_off + cout].any(), "conv writes a channel twice"
        d = ConvDesc(i, in_off, o, out_off, res, res_off, bcast, cin, cout, k, s, relu, up, norm, pw, engine)
        fan = cin * TAPS[k] if k != 42 else 4 * cin
        shape = (cin, cout, 4, 4) if k == 42 else (cout, cin * TAPS[k])
        w = bf16_round(self.rng.standard_normal(shape) * (1.2 / math.sqrt(fan))).reshape(-1)
        if self.tensors[i]["dt"] == U8 and not norm:      # raw 0..255 values
            w = bf16_round(w / 128.0)
        b = (0.1 * self.rng.standard_normal(cout)).astype(np.float32)
        if self.rng.random() < 0.15 and not self.tensors[o]["nchw"]:
            b = None
        op = self._op(("conv", (d, w, b)), lane)
        self.written[o][out_off:out_off + cout] = True
        return op

    def sum(self, out, base, terms, ups, offs, relu=1, lane=0):
        Cc = self.tensors[out]["C"]
        assert self.written[base].all() and not self.written[out].any()
        for t, o in zip(terms, offs):
            assert self.written[t][o:o + Cc].all()
        n = len(terms)
        s = SumDesc(out, base, n, (C.c_int * 4)(*(list(terms) + [0] * (4 - n))), (C.c_int * 4)(*(list(ups) + [1] * (4 - n))),
                    relu, (C.c_int * 4)(*(list(offs) + [0] * (4 - n))))
        op = self._op(("sum", (s,)), lane)
        self.written[out][:] = True
        return op

    def maxpool(self, i, o, lane=0):
        assert self.written[i].all() and not self.written[o].any()
        op = self._op(("maxpool", (i, o)), lane)
        self.written[o][:] = True
        return op

    def _op(self, call, lane):
        op = self.n_ops
        self.n_ops += 1
        self.calls.append((call[0], op, call[1]))
        if lane:
            self.calls.append(("lane", None, (op, lane)))
        self.lanes[op] = lane
        return op

    def record(self):
        return dict(calls=self.calls, tensors=self.tensors, max_batch=self.batch)

    # ---- helpers ---------------------------------------------------------------------------------------------------
    def pick(self, seq):
        return seq[int(self.rng.integers(len(seq)))]

    def lane(self):
        return int(self.rng.integers(4)) if self.rng.random() < 0.5 else 0

    def ext_input(self, H, W, dt, Cc=16):
        key = (H, W, dt, Cc)
        if key not in self.ext_in:
            t = self.tensor(H, W, Cc, dt, ext=1)
            self.written[t][:] = True
            self.inputs.append(t)
            self.ext_in[key] = t
        return self.ext_in[key]

    def feed(self, H, W, Cc, dt, relu=1):
        """a new internal NHWC tensor written whole by a 1x1 conv of an external input (SIMT: external input)"""
        src = self.ext_input(H, W, F32 if dt == F32 else BF16)
        t = self.tensor(H, W, Cc, dt)
        self.conv(src, t, 16, Cc, k=1, relu=relu, lane=self.lane())
        self.pool.append(t)
        return t

    def source(self, H, W, cin, dt, whole=False):
        """(tensor, in_c_off) of an internal tensor written whole with >= cin channels at H x W: from the pool or fed"""
        if not whole:
            cands = [t for t in self.pool if (self.tensors[t]["H"], self.tensors[t]["W"], self.tensors[t]["dt"]) == (H, W, dt)
                     and self.tensors[t]["C"] >= cin]
            if cands and self.rng.random() < 0.6:
                t = self.pick(cands)
                offs = list(range(0, self.tensors[t]["C"] - cin + 1, 8))
                return t, self.pick(offs)
        extra = self.pick((0, 0, 0, 16, 32)) if not whole else 0
        t = self.feed(H, W, cin + extra, dt)
        return t, self.pick((0, extra)) if extra else 0

    def output(self, H, W, cout, dt, fill_from=None):
        """(tensor, out_c_off) of a fresh NHWC output; with spare channels a second op writes the rest of the tensor
        (skip-concat style) from fill_from = (tensor, c_off, cin)"""
        extra = self.pick((0, 0, 16, 32)) if fill_from is not None else 0
        t = self.tensor(H, W, cout + extra, dt)
        off = self.pick((0, extra)) if extra else 0
        return t, off

    def fill_rest(self, t, src, src_off, cin):
        """write the channels of t still unwritten with a 1x1 conv of src's slice (same resolution)"""
        free = np.flatnonzero(~self.written[t])
        if len(free):
            self.conv(src, t, cin, len(free), k=1, in_off=src_off, out_off=int(free[0]), relu=1, lane=self.lane())
        self.pool.append(t)

    def residual(self, H, W, cout, dt_allowed):
        """(res, res_c_off, broadcast) of a residual at H x W, or (-1, 0, 0)"""
        r = self.rng.random()
        if r < 0.45:
            return -1, 0, 0
        if r < 0.6 and F32 in dt_allowed:
            return self.const(H, W, cout), 0, 1
        t, off = self.source(H, W, cout, self.pick(dt_allowed))
        return t, off, 0

    def expect_op(self, item, ops, plan):
        self.expect.append((item, tuple(ops), plan))


# ---- planted items ---------------------------------------------------------------------------------------------------
MODE_KS = {1: (1, 1), 3: (3, 1), 2: (3, 2)}


def plant_tc(g, mode, cin, nt, eb, generic):
    """one conv on B2R_CASE row (mode, cin, nt, eb), in the direct-NHWC or the generic epilogue instantiation"""
    k, s = MODE_KS[mode]
    dt = BF16 if eb == 2 else F32
    engine = (ENGINE_AUTO if g.rng.random() < 0.7 else ENGINE_WGMMA) if eb == 2 else ENGINE_TF32
    if nt == 16:
        cout = g.pick((32, 64))
    elif nt == 32:
        cout = g.pick((32, 96))
    else:
        cout = g.pick((64, 192, 256)) if (mode, cin, eb) == (3, 128, 2) else g.pick((64, 128))
    Ho = g.pick((16, 32)) if mode == 2 else g.pick((16, 32, 48, 64))
    Wo = g.pick((16, 24, 32)) if mode == 2 else g.pick((16, 24, 32, 48, 64))
    if (mode, cin, eb, cout) == (3, 32, 2, 32):
        Wo = g.pick((24, 40, 56))         # W % 16 != 0: not the pixel-pair fold
    H, W = (2 * Ho, 2 * Wo) if mode == 2 else (Ho, Wo)
    lane = g.lane()
    up, nchw, pw = 1, 0, -1
    if generic:
        if mode != 2 and g.rng.random() < 0.5:
            nchw = 1
            cout = 35 if nt == 32 else (64 if nt == 64 else 32)
            pw = 0 if g.rng.random() < 0.5 else -1
        else:
            up = 2
    if not generic and mode != 2 and g.rng.random() < 0.25:
        # output slice in the input's own tensor: [0, cin) read, [cin, cin + cout) written
        x = g.tensor(H, W, cin + cout, dt)
        src = g.ext_input(H, W, dt)
        g.conv(src, x, 16, cin, k=1, lane=g.lane())
        res, roff, bc = g.residual(Ho, Wo, cout, (F32,) if eb == 4 else (BF16, F32))
        op = g.conv(x, x, cin, cout, k, s, 0, cin, res, roff, bc, relu=int(g.rng.random() < 0.7), engine=engine, lane=lane)
        g.pool.append(x)
    else:
        x, xoff = g.source(H, W, cin, dt)
        if nchw:
            o, ooff = g.tensor(Ho, Wo, cout, F32, nchw=1, ext=1), 0
            res, roff, bc = -1, 0, 0
        else:
            o, ooff = g.output(Ho * up, Wo * up, cout, dt, fill_from=x)
            res, roff, bc = g.residual(Ho * up, Wo * up, cout, (F32,) if eb == 4 else (BF16, F32))
        op = g.conv(x, o, cin, cout, k, s, xoff, ooff, res, roff, bc, relu=int(g.rng.random() < 0.7 and pw < 0), up=up,
                    pw=pw, engine=engine, lane=lane)
        if not nchw:
            if up == 1 and mode != 2:
                g.fill_rest(o, x, xoff, cin)
            else:
                _fill_any(g, o)
    g.expect_op(f"tc row {mode}/{cin}/{nt}/{'bf16' if eb == 2 else 'tf32'} {'generic' if generic else 'direct'}", [op],
                ("tc", (mode, cin, nt, eb, generic)))


def _fill_any(g, t):
    """write t's unwritten channels with a 1x1 SIMT conv of a fed tensor at its resolution"""
    free = np.flatnonzero(~g.written[t])
    if len(free):
        T = g.tensors[t]
        src = g.ext_input(T["H"], T["W"], F32 if T["dt"] == F32 else BF16)
        g.conv(src, t, 16, len(free), k=1, out_off=int(free[0]), lane=g.lane())
    g.pool.append(t)


def plant_swap(g):
    side = g.pick((32, 64))
    x, xoff = g.source(side, side, 128, BF16)
    o = g.tensor(side, side, 128, BF16)
    res, roff, bc = g.residual(side, side, 128, (BF16, F32))
    op = g.conv(x, o, 128, 128, 3, 1, xoff, 0, res, roff, bc, lane=g.lane())
    g.pool.append(o)
    g.expect_op("SWAP 128->128 (kind 31)", [op], ("kind", 31))


def plant_stream(g):
    """64x64 frames: 16 tiles of 16x16 per 64-channel slab, so the graph batch gives some CTA 3 work items"""
    cout = g.pick((64, 128, 256))
    x, xoff = g.source(64, 64, 256, BF16)
    o = g.tensor(64, 64, cout, BF16)
    res, roff, bc = g.residual(64, 64, cout, (BF16, F32))
    op = g.conv(x, o, 256, cout, 3, 1, xoff, 0, res, roff, bc, lane=g.lane())
    g.pool.append(o)
    g.expect_op("streamed 256->64k (kind 34)", [op], ("kind", 34))


def plant_stem(g):
    src = g.tensor(128, 128, 3, U8, ext=1)
    g.written[src][:] = True
    g.inputs.append(src)
    o = g.tensor(64, 64, 64, BF16)
    op = g.conv(src, o, 3, 64, 3, 2, norm=1, lane=g.lane())
    g.pool.append(o)
    g.expect_op("stem u8 3->64 (kind 33)", [op], ("kind", 33))


def plant_conv1d(g):
    x, xoff = g.source(16, 128, g.pick((64, 128)), BF16, whole=True)
    cin = g.tensors[x]["C"]
    cout = g.pick((32, 64))
    o = g.tensor(16, 128, cout, BF16)
    res, roff, bc = g.residual(16, 128, cout, (BF16,))
    op = g.conv(x, o, cin, cout, 13, 1, 0, 0, res, roff, bc, relu=1, lane=g.lane())
    g.pool.append(o)
    g.expect_op("Conv1d (kind 13)", [op], ("kind", 13))


def plant_k7(g):
    if g.rng.random() < 0.5:
        src = g.tensor(64, 64, 3, U8, ext=1)
        g.written[src][:] = True
        g.inputs.append(src)
        cin, dt, off = 3, BF16, 0
    else:
        src, off = g.source(32, 32, 16, g.pick((BF16, F32)))
        cin, dt = 16, g.tensors[src]["dt"]
    H, W = g.tensors[src]["H"], g.tensors[src]["W"]
    s = g.pick((1, 2))
    Ho, Wo = out_hw(7, s, H, W)
    cout = g.pick((16, 32, 64))
    o = g.tensor(Ho, Wo, cout, dt)
    bias_map = g.const(Ho, Wo, cout) if g.rng.random() < 0.5 else -1
    op = g.conv(src, o, cin, cout, 7, s, off, 0, bias_map, 0, int(bias_map >= 0), lane=g.lane())
    g.pool.append(o)
    g.expect_op("Generic7x7", [op], ("simt", "k7"))


def plant_deconv(g):
    side = g.pick((8, 16, 32))
    dt = g.pick((BF16, F32))
    x, xoff = g.source(side, side, g.pick((16, 32, 64)), dt)
    cin = g.tensors[x]["C"] - xoff if g.rng.random() < 0.3 else 16
    cin = min(cin, g.tensors[x]["C"] - xoff)
    cout = g.pick((16, 32))
    o = g.tensor(2 * side, 2 * side, cout, dt)
    op = g.conv(x, o, cin, cout, 42, 2, xoff, 0, lane=g.lane())
    g.pool.append(o)
    g.expect_op("Deconv4x4", [op], ("simt", "deconv"))


def plant_simt(g, inst):
    """the SIMT instantiations: conv_stem_kernel, conv_simt_kernel<1,3,1>, <3,3,1>, <3,3,2>, <1,1,1>, <1,1,2>"""
    if inst == "stem":
        src = g.ext_input(64, 64, U8, 3)
        o = g.tensor(32, 32, 32, BF16)
        op = g.conv(src, o, 3, 32, 3, 2, norm=1, lane=g.lane())
        g.pool.append(o)
    else:
        k, s = {"131": (13, 1), "331": (3, 1), "332": (3, 2), "111": (1, 1), "112": (1, 2)}[inst]
        dt = g.pick((F32, BF16))
        engine = ENGINE_AUTO if dt == F32 else ENGINE_SIMT
        H = g.pick((16, 24, 32))
        W = 128 if k == 13 and g.rng.random() < 0.5 else g.pick((16, 24, 32))
        cin = g.pick((8, 16, 24, 32, 48, 64))
        x, xoff = g.source(H, W, cin, dt)
        Ho, Wo = out_hw(k, s, H, W)
        cout = g.pick((8, 16, 24, 35, 64)) if k != 13 else g.pick((16, 32))
        up = g.pick((1, 1, 2)) if k != 13 else 1
        if g.rng.random() < 0.3 and k != 13:
            o = g.tensor(Ho * up, Wo * up, cout, F32, nchw=1, ext=1)
            op = g.conv(x, o, cin, cout, k, s, xoff, 0, relu=0, up=up, pw=0 if g.rng.random() < 0.5 else -1,
                        engine=engine, lane=g.lane())
        else:
            odt = g.pick((F32, BF16))
            o = g.tensor(Ho * up, Wo * up, cout, odt)
            res, roff, bc = g.residual(Ho * up, Wo * up, cout, (BF16, F32))
            op = g.conv(x, o, cin, cout, k, s, xoff, 0, res, roff, bc, relu=int(g.rng.random() < 0.6), up=up,
                        engine=engine, lane=g.lane())
            g.pool.append(o)
    g.expect_op(f"SIMT {inst}", [op], ("simt", inst))


def plant_maxpool(g, dt):
    H, W = g.pick((16, 24, 32)), g.pick((16, 24, 32, 40))
    x, _ = g.source(H, W, g.pick((8, 16, 32)), dt, whole=True)
    o = g.tensor((H - 1) // 2 + 1, (W - 1) // 2 + 1, g.tensors[x]["C"], dt)
    op = g.maxpool(x, o, lane=g.lane())
    g.pool.append(o)
    g.expect_op(f"maxpool {'bf16' if dt == BF16 else 'fp32'}", [op], ("maxpool", dt))


def plant_sum(g, kernel, dt):
    """a fuse-sum the default selection runs on `kernel`: pipe when every tensor has the base's dtype and a row has
    >= 128 8-channel chunks (<= 16 KiB), else simple"""
    if kernel == "pipe":
        H, W, Cc = g.pick((16, 32)), 64, g.pick((16, 32, 64))
    else:
        H, W, Cc = g.pick((16, 32)), g.pick((16, 32)), g.pick((8, 16, 32))
    base, _ = g.source(H, W, Cc, dt, whole=True)
    n = int(g.rng.integers(1, 5))
    terms, ups, offs = [], [], []
    for _ in range(n):
        u = g.pick([u for u in (1, 2, 4, 8) if H % u == 0 and W % u == 0 and H // u >= 2])
        tdt = dt if kernel == "pipe" else g.pick((BF16, F32))
        extra = g.pick((0, 0, 8, 16))
        t = g.feed(H // u, W // u, Cc + extra, tdt)
        terms.append(t)
        ups.append(u)
        offs.append(g.pick((0, extra)))
    odt = dt if kernel == "pipe" else g.pick((BF16, F32))
    if kernel == "simple" and all(g.tensors[t]["dt"] == dt for t in terms) and odt == dt and W * Cc // 8 >= 128:
        odt = BF16 if dt == F32 else F32
    o = g.tensor(H, W, Cc, odt)
    op = g.sum(o, base, terms, ups, offs, relu=int(g.rng.random() < 0.7), lane=g.lane())
    g.pool.append(o)
    g.expect_op(f"fuse-sum {kernel} {'bf16' if dt == BF16 else 'fp32'}", [op], ("sum", kernel))


def plant_block(g, fold, variant=None):
    """relu(conv2(relu(conv1(x))) + x), 3x3 64->64 (or pixel-pair foldable 32->32) on 64x64 frames; a near-miss variant
    keeps the two convs apart"""
    Cc = 32 if fold else 64
    H = W = 64
    if variant == "odd side":
        H, W = 56, 56
    lane = g.lane()
    if fold or g.rng.random() < 0.5:
        x = g.feed(H, W, Cc, BF16)
        xoff = 0
    else:
        x = g.feed(H, W, 2 * Cc, BF16)
        xoff = g.pick((0, Cc))
    t = g.tensor(H, W, Cc, BF16, ext=int(variant == "intermediate external"))
    a = g.conv(x, t, Cc, Cc, 3, 1, xoff, 0, relu=int(variant != "no ReLU"), lane=lane)
    if variant == "second reader":
        r2 = g.tensor(H, W, 16, BF16)
        g.conv(t, r2, Cc, 16, 1, lane=lane)
        g.pool.append(r2)
    if fold:
        y, yoff = g.tensor(H, W, Cc, BF16), 0
    else:
        y = g.tensor(H, W, g.pick((Cc, 2 * Cc)), BF16)
        yoff = g.pick((0, g.tensors[y]["C"] - Cc))
    if variant == "residual from another slice":
        x2 = x if g.tensors[x]["C"] == 2 * Cc else g.feed(H, W, 2 * Cc, BF16)
        res, roff = x2, (Cc if (x2 != x or xoff == 0) else 0)
    else:
        res, roff = x, xoff
    b = g.conv(t, y, Cc, Cc, 3, 1, 0, yoff, res, roff, lane=(lane + 1) % 4 if variant == "different lanes" else lane)
    _fill_any(g, y)
    if variant is None:
        g.expect_op(f"block {'folded' if fold else '64'}", [a, b], ("block", fold))
    else:
        g.expect_op(f"block near miss: {variant}", [a, b], ("unfused",))


def plant_bottleneck(g, stored, variant=None):
    """relu(conv3(relu(conv2(relu(conv1(x))))) + x): 1x1 256->64, 3x3 64->64, 1x1 64->256 on 64x64 frames"""
    lane = g.lane()
    x = g.feed(64, 64, 256, BF16)
    t1 = g.tensor(64, 64, 64, BF16, ext=int(variant == "intermediate external"))
    t2 = g.tensor(64, 64, 64, BF16)
    a = g.conv(x, t1, 256, 64, 1, 1, lane=lane)
    b = g.conv(t1, t2, 64, 64, 3, 1, relu=int(variant != "no ReLU"), lane=lane)
    y = g.tensor(64, 64, 256, BF16)
    c = g.conv(t2, y, 64, 256, 1, 1, 0, 0, x, 0, lane=(lane + 1) % 4 if variant == "different lanes" else lane)
    g.pool.append(y)
    if stored:
        for t in ([t1] if stored == 1 else [t2] if stored == 2 else [t1, t2]):
            r = g.tensor(64, 64, 16, BF16)
            g.conv(t, r, 64, 16, 1, lane=g.lane())
            g.pool.append(r)
    if variant is None:
        g.expect_op(f"bottleneck {'stored t' + str(stored) if stored else 'unstored'}", [a, b, c], ("bottleneck", bool(stored)))
    else:
        g.expect_op(f"bottleneck near miss: {variant}", [a, b, c], ("unfused",))


def plant_fallback(g, what):
    """a conv one step outside a tensor-core condition: it must run on the SIMT engine"""
    dt, engine = BF16, ENGINE_AUTO
    H, W, cin, cout, k, s, xoff, up = 32, 32, 64, 64, 3, 1, 0, 1
    res_dt = None
    if what == "cin 48":
        cin = 48
    elif what == "cout 48":
        cout = 48
    elif what == "height 40":
        H = 40
    elif what == "width 20":
        W = 20
    elif what == "stride-2 height 24":
        H, s = 24, 2
    elif what == "in_c_off 4":
        xoff = 4
    elif what == "tf32 with bf16 residual":
        dt, engine, res_dt = F32, ENGINE_TF32, BF16
    elif what == "tf32 256-channel stride 2":
        dt, engine, cin, s = F32, ENGINE_TF32, 256, 2
    if what == "external input":
        x = g.ext_input(H, W, dt, cin)
    elif xoff:
        x = g.feed(H, W, cin + 8, dt)
    else:
        x, xoff = g.source(H, W, cin, dt)
    Ho, Wo = out_hw(k, s, H, W)
    o = g.tensor(Ho * up, Wo * up, cout, dt)
    res, roff = -1, 0
    if res_dt is not None:
        res = g.feed(Ho, Wo, cout, res_dt)
    op = g.conv(x, o, cin, cout, k, s, xoff, 0, res, roff, lane=g.lane(), engine=engine)
    g.pool.append(o)
    g.expect_op(f"SIMT fallback: {what}", [op], ("simt", f"{k}{k}{s}"))


def items():
    """every planted item: (name, plant function)"""
    import os
    src = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "romp_b200", "csrc", "conv_tc.cu")).read()
    rows = b2r_rows(src)
    dead = set(unreachable_rows(rows))
    out = []
    for row in rows:
        if row in dead:
            continue
        for generic in (False, True):
            out.append((row, generic))
    its = [(f"tc {r} {'generic' if gen else 'direct'}", (lambda r=r, gen=gen: lambda g: plant_tc(g, *r, gen))()) for r, gen in out]
    its += [("swap", plant_swap), ("stream", plant_stream), ("stem", plant_stem), ("conv1d", plant_conv1d), ("k7", plant_k7),
            ("deconv", plant_deconv)]
    its += [(f"simt {i}", (lambda i=i: lambda g: plant_simt(g, i))()) for i in ("stem", "131", "331", "332", "111", "112")]
    its += [(f"maxpool {dt}", (lambda dt=dt: lambda g: plant_maxpool(g, dt))()) for dt in (BF16, F32)]
    its += [(f"sum {k} {dt}", (lambda k=k, dt=dt: lambda g: plant_sum(g, k, dt))()) for k, dt in
            (("pipe", BF16), ("pipe", F32), ("simple", BF16), ("simple", F32))]
    its += [("block 64", lambda g: plant_block(g, False)), ("block folded", lambda g: plant_block(g, True))]
    its += [(f"bottleneck stored {s}", (lambda s=s: lambda g: plant_bottleneck(g, s))()) for s in (0, 1, 2, 3)]
    for v in ("intermediate external", "second reader", "different lanes", "residual from another slice", "no ReLU",
              "odd side"):
        its.append((f"block near miss {v}", (lambda v=v: lambda g: plant_block(g, False, v))()))
    for v in ("intermediate external", "different lanes", "no ReLU"):
        its.append((f"bottleneck near miss {v}", (lambda v=v: lambda g: plant_bottleneck(g, 0, v))()))
    for w in ("cin 48", "cout 48", "height 40", "width 20", "stride-2 height 24", "in_c_off 4", "tf32 with bf16 residual",
              "tf32 256-channel stride 2", "external input"):
        its.append((f"fallback {w}", (lambda w=w: lambda g: plant_fallback(g, w))()))
    return its


def planted_items(seed, n_items, n_seeds):
    """the items seed plants: an even share of all of them, so that SEEDS covers each once"""
    per = -(-n_items // n_seeds)
    return [(seed * per + j) % n_items for j in range(per)]


# ---- random ops ------------------------------------------------------------------------------------------------------
def random_op(g):
    r = g.rng.random()
    if r < 0.6:
        cands = [t for t in g.pool if g.tensors[t]["H"] <= 64]
        if not cands:
            return
        x = g.pick(cands)
        T = g.tensors[x]
        k = g.pick((1, 1, 3, 3, 7, 13, 42))
        s = g.pick((1, 2)) if k in (1, 3, 7) else (2 if k == 42 else 1)
        cin = g.pick([c for c in (8, 16, 24, 32, 48, 64, 96, 128, 192, 256) if c <= T["C"]] or [T["C"]])
        xoff = g.pick(list(range(0, T["C"] - cin + 1, 8)) or [0])
        Ho, Wo = out_hw(k, s, T["H"], T["W"])
        up = g.pick((1, 1, 1, 2, 4)) if k not in (13, 42) else 1
        if Ho * up > 128 or Wo * up > 128:
            up = 1
        cout = g.pick((8, 16, 24, 32, 48, 64, 96, 128))
        if T["dt"] == F32:
            engine = g.pick((ENGINE_AUTO, ENGINE_TF32, ENGINE_SIMT))
        else:
            engine = g.pick((ENGINE_AUTO, ENGINE_AUTO, ENGINE_SIMT))
        if g.rng.random() < 0.2 and k != 13:
            o = g.tensor(Ho * up, Wo * up, cout, F32, nchw=1, ext=1)
            g.conv(x, o, cin, cout, k, s, xoff, 0, relu=0, up=up, pw=g.pick((-1, 0)), engine=engine, lane=g.lane())
            return
        odt = g.pick((T["dt"], T["dt"], BF16, F32))
        o, ooff = g.output(Ho * up, Wo * up, cout, odt, fill_from=x)
        res, roff, bc = g.residual(Ho * up, Wo * up, cout, (BF16, F32))
        g.conv(x, o, cin, cout, k, s, xoff, ooff, res, roff, bc, relu=int(g.rng.random() < 0.6), up=up, engine=engine,
               lane=g.lane())
        _fill_any(g, o)
    elif r < 0.85:
        cands = [t for t in g.pool if g.tensors[t]["C"] % 8 == 0]
        if not cands:
            return
        base = g.pick(cands)
        B = g.tensors[base]
        n = int(g.rng.integers(1, 5))
        terms, ups, offs = [], [], []
        for _ in range(n):
            us = [u for u in (1, 2, 4, 8) if B["H"] % u == 0 and B["W"] % u == 0]
            u = g.pick(us)
            tc = [t for t in g.pool if g.tensors[t]["H"] * u == B["H"] and g.tensors[t]["W"] * u == B["W"] and
                  g.tensors[t]["C"] % 8 == 0 and g.tensors[t]["C"] >= B["C"] and g.tensors[t]["dt"] != U8]
            if tc and g.rng.random() < 0.7:
                t = g.pick(tc)
                off = g.pick(list(range(0, g.tensors[t]["C"] - B["C"] + 1, 8)))
            else:
                extra = g.pick((0, 8))
                t = g.feed(B["H"] // u, B["W"] // u, B["C"] + extra, g.pick((BF16, F32)))
                off = g.pick((0, extra))
            terms.append(t)
            ups.append(u)
            offs.append(off)
        o = g.tensor(B["H"], B["W"], B["C"], g.pick((BF16, F32)))
        g.sum(o, base, terms, ups, offs, relu=int(g.rng.random() < 0.5), lane=g.lane())
        g.pool.append(o)
    else:
        cands = [t for t in g.pool if g.tensors[t]["dt"] != U8 and g.tensors[t]["H"] >= 8]
        if not cands:
            return
        x = g.pick(cands)
        T = g.tensors[x]
        o = g.tensor((T["H"] - 1) // 2 + 1, (T["W"] - 1) // 2 + 1, T["C"], T["dt"])
        g.maxpool(x, o, lane=g.lane())
        g.pool.append(o)


def finish(g):
    """one external output per seed that sums nothing up: a 1x1 conv of the last pooled tensor into an external NHWC
    tensor, so that every graph has an NHWC output the bit comparisons read"""
    x = g.pool[-1]
    T = g.tensors[x]
    o = g.tensor(T["H"], T["W"], 8, g.pick((BF16, F32)), ext=1)
    g.conv(x, o, min(T["C"], 64), 8, 1, lane=g.lane())


_ITEMS = None


def generate(seed, n_seeds=len(SEEDS)):
    """-> Graph of `seed`: its planted items, then random ops over everything written"""
    global _ITEMS
    if _ITEMS is None:
        _ITEMS = items()
    g = Graph(seed)
    picks = planted_items(seed, len(_ITEMS), n_seeds)
    g.items = [_ITEMS[i][0] for i in picks]
    for i in picks:
        _ITEMS[i][1](g)
        for _ in range(int(g.rng.integers(0, 2))):
            random_op(g)
    for _ in range(int(g.rng.integers(2, 6))):
        random_op(g)
    finish(g)
    return g


# ---------------------------------------------------------------------------------------------------------------------
# the library's rules, restated
# ---------------------------------------------------------------------------------------------------------------------
def _overlap(a, n, b, m):
    return a < b + m and b < a + n


def aliasing_violations(r):
    """ops of record r that break the aliasing rule of include/b200romp.h: a slice read of the output tensor overlaps the
    output slice without being it (identical slices only for an elementwise read: a batched residual, a sum base or an
    up-1 term); a maxpool of its own output"""
    bad = []
    for kind, op, args in r["calls"]:
        if kind == "conv":
            d = args[0]
            if d.in_ == d.out and _overlap(d.in_c_off, d.cin, d.out_c_off, d.cout):
                bad.append(f"op {op}: input overlaps the output slice")
            if d.res == d.out and _overlap(d.res_c_off, d.cout, d.out_c_off, d.cout) and (
                    d.res_c_off != d.out_c_off or d.res_broadcast):
                bad.append(f"op {op}: residual overlaps the output slice")
        elif kind == "sum":
            s = args[0]
            for k in range(s.n_terms):
                if s.term[k] == s.out and (s.up[k] != 1 or s.term_c_off[k] != 0):
                    bad.append(f"op {op}: sum term {k} overlaps the output")
        elif kind == "maxpool" and args[0] == args[1]:
            bad.append(f"op {op}: maxpool in place")
    return bad


def check_record(r):
    """-> list of violations of the rules in the module docstring (empty: the graph is valid)"""
    T = r["tensors"]
    bad = []
    written = {t: np.zeros(s["C"], bool) for t, s in T.items()}
    # external inputs: external tensors no op writes, bound whole by the caller
    outs_all = {a[0].out for k, _, a in r["calls"] if k == "conv"} | {a[0].out for k, _, a in r["calls"] if k == "sum"} | {
        a[1] for k, _, a in r["calls"] if k == "maxpool"}
    for t, s in T.items():
        if s["const"] or (s["ext"] and t not in outs_all):
            written[t][:] = True
    # the generator keeps even the identical-slice forms out: each channel is written once
    bad += aliasing_violations(r)

    def readable(t, lo, n):
        return bool(written[t][lo:lo + n].all())

    for kind, op, args in r["calls"]:
        if kind == "conv":
            d = args[0]
            ti, to = T[d.in_], T[d.out]
            if d.ksize not in (1, 3, 7, 13, 42) or d.stride not in (1, 2) or d.upsample not in (1, 2, 4, 8):
                bad.append(f"op {op}: ksize/stride/upsample")
            if (d.ksize == 13 and (d.stride != 1 or d.upsample != 1)) or (d.ksize == 42 and (d.stride != 2 or d.upsample != 1)):
                bad.append(f"op {op}: ksize code with stride/upsample")
            if ti["nchw"] or not (d.cin > 0 and 0 <= d.in_c_off and d.in_c_off + d.cin <= ti["C"]):
                bad.append(f"op {op}: input slice")
            if not (d.cout > 0 and 0 <= d.out_c_off and d.out_c_off + d.cout <= to["C"]):
                bad.append(f"op {op}: output slice")
            Ho, Wo = out_hw(d.ksize, d.stride, ti["H"], ti["W"])
            if (Ho * d.upsample, Wo * d.upsample) != (to["H"], to["W"]):
                bad.append(f"op {op}: output shape")
            if ti["dt"] == U8 and not (d.input_norm or d.ksize == 7):
                bad.append(f"op {op}: u8 input")
            if to["dt"] == U8 or (to["nchw"] and to["dt"] != F32) or to["const"]:
                bad.append(f"op {op}: output dtype")
            if to["nchw"] and not to["ext"]:
                bad.append(f"op {op}: internal NCHW output")
            if d.res >= 0:
                tr = T[d.res]
                if (tr["H"], tr["W"]) != (to["H"], to["W"]) or tr["nchw"] or tr["dt"] == U8 or not (
                        0 <= d.res_c_off and d.res_c_off + d.cout <= tr["C"]):
                    bad.append(f"op {op}: residual")
                if d.res_broadcast and not tr["const"]:
                    bad.append(f"op {op}: broadcast residual is not a const tensor")
                if not readable(d.res, d.res_c_off, d.cout):
                    bad.append(f"op {op}: residual read before written")
            if not readable(d.in_, d.in_c_off, d.cin):
                bad.append(f"op {op}: input read before written")
            if d.pow_channel >= d.cout:
                bad.append(f"op {op}: pow channel")
            outs = [(d.out, d.out_c_off, d.cout)]
        elif kind == "sum":
            s = args[0]
            to, tb = T[s.out], T[s.base]
            if to["nchw"] or tb["nchw"] or U8 in (to["dt"], tb["dt"]) or to["C"] % 8 or (tb["H"], tb["W"], tb["C"]) != (
                    to["H"], to["W"], to["C"]) or not 1 <= s.n_terms <= 4:
                bad.append(f"op {op}: sum base/out")
            if s.base == s.out or not readable(s.base, 0, to["C"]):
                bad.append(f"op {op}: sum base")
            for k in range(s.n_terms):
                tt, u, co = T[s.term[k]], s.up[k], s.term_c_off[k]
                if u not in (1, 2, 4, 8) or tt["nchw"] or tt["dt"] == U8 or tt["C"] % 8 or co % 8 or co + to["C"] > tt["C"] or (
                        tt["H"] * u, tt["W"] * u) != (to["H"], to["W"]):
                    bad.append(f"op {op}: sum term {k}")
                if s.term[k] == s.out or not readable(s.term[k], co, to["C"]):
                    bad.append(f"op {op}: sum term {k} read")
            outs = [(s.out, 0, to["C"])]
        elif kind == "maxpool":
            i, o = args
            ti, to = T[i], T[o]
            if ti["nchw"] or to["nchw"] or ti["dt"] != to["dt"] or ti["dt"] == U8 or ti["C"] != to["C"] or i == o or (
                    to["H"], to["W"]) != ((ti["H"] - 1) // 2 + 1, (ti["W"] - 1) // 2 + 1):
                bad.append(f"op {op}: maxpool")
            if not readable(i, 0, ti["C"]):
                bad.append(f"op {op}: maxpool input read before written")
            outs = [(o, 0, to["C"])]
        else:
            continue
        for t, lo, n in outs:
            if written[t][lo:lo + n].any():
                bad.append(f"op {op}: writes channels of tensor {t} twice")
            written[t][lo:lo + n] = True
    return bad


# ---------------------------------------------------------------------------------------------------------------------
# the buffer planner of b200romp_net_finalize, on describe()'s op list
# ---------------------------------------------------------------------------------------------------------------------
def plan_workspace(tensors, ops, max_batch):
    """ops: per describe() op, dict(reads=[tensor ids], writes=[tensor ids], lane).  -> (total bytes, buffers), buffers =
    per buffer the list of (tensor, writer op index) it holds in allocation order"""
    first_def, last_use = {}, {}
    for i, op in enumerate(ops):
        for t in op["writes"]:
            first_def.setdefault(t, i)
            last_use[t] = max(last_use.get(t, -1), i)
        for t in op["reads"]:
            last_use[t] = max(last_use.get(t, -1), i)
    dies = {}
    for t in sorted(tensors):
        s = tensors[t]
        if not s["ext"] and not s["const"] and t in first_def:
            dies.setdefault(last_use[t], []).append(t)
    free, bufs, tbuf, total = {}, [], {}, 0
    for i, op in enumerate(ops):
        for t in op["writes"]:
            s = tensors[t]
            if s["ext"] or s["const"] or first_def[t] != i:
                continue
            nb = (s["H"] * s["W"] * s["C"] * DSIZE[s["dt"]] * max_batch + 1023) // 1024 * 1024
            if free.get(nb):
                b = free[nb].pop(0)
            else:
                bufs.append(dict(bytes=nb, held=[]))
                b = len(bufs) - 1
                total += nb
            tbuf[t] = b
            bufs[b]["held"].append((t, i))
        for t in dies.get(i, []):
            free.setdefault(bufs[tbuf[t]]["bytes"], []).append(tbuf[t])
    return total, bufs
