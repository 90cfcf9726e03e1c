"""Every conv graph the builder emits computes the model it claims to, checked whole in float64 without a GPU.

test_gpu_graph_ops checks each op of a built graph against float64 from the tensors that op read and the weights it was
given.  That takes the wiring (which tensor, channel slice and residual an op reads) and the rewritten weights as given.
This file checks the program itself: graph.py runs against FakeLib, a stand-in for the library that numbers tensors and
ops as the library does, and the Recorder of test_gpu_graph_ops copies every call.  The record is then interpreted op by
op in float64 (the per-op references of test_gpu_graph_ops: conv_linear, normalise_input, pow_f32_11, sum_terms,
maxpool_ref) and compared with the float64 oracle of the model (oracle/romp_oracle.py, oracle/bev_oracle.py) on one
synthetic u8 frame with the seeded synthetic weights.  graph.round_bf16 is the identity while recording, so a bf16 graph
is interpreted with its unrounded folded weights; test_bf16_rounding checks the rounding on its own.

The bound.  Every op is computed twice: on its input values, giving v, and on |x|, |W|, |b|, |res| (a sum: |base| + the
|terms|), giving A, the magnitude that op summed its output from, as conv_bound and sum_bound do; on the pow channel
A = 1.1^z A_z (d 1.1^z = ln 1.1 1.1^z dz), and a maxpool passes on the largest A of its window.  (A carried through the
graph as |W| A_in instead grows about 12x per 3x3 layer, and 10^100 over the graph: no bound at all.)  Every element must
satisfy |v - ref| <= 2^-18 A.  Between the two float64 computations the only rounding is the builder's: each folded
weight and bias is the fp32 cast of a float64 BN fold (relative error <= 2^-24, at most 2^-24 A per layer), and a few
constant folds are computed in fp32 (the head and stem bias maps, b3 + bd).  These independent roundings add along a path
like a random walk, about sqrt(L) 2^-24 of the activations after L convs; the longest path is 99 convs (ROMP HRNet to the
heads, printed per output), so 2^-18 = 64 x 2^-24 is 6x sqrt(99) 2^-24.  Measured: the worst |v - ref| / (2^-18 A) is
0.005 - 0.07 over the matrix (printed per output).  A wiring error moves elements by a sizeable fraction of A, 2^18 times
the bound: the negative controls below are rejected by ratios of 1.5e3 - 2.3e5 (they must exceed 100).

Matrix (the same record, i.e. the same op list, descriptors without the engine, tensor shapes and weight bytes, is
interpreted once; records differ only where a rewrite differs):
  ROMP HRNet {fp32, tf32, bf16} x {default, B200ROMP_NO_SKIP_CONCAT=1, B200ROMP_NO_FUSE1X1_MERGE=1}: backbone_out,
      center_maps, params_maps.  Rewrites: input_norm on the first conv; the layer1.0 skip concat ([W3 | Wd] over a
      128-channel tensor written at out_c_off 0 and 64, bias b3 + bd; not with NO_SKIP_CONCAT); the merged 1x1 fuse convs
      (output channels zero-padded to a multiple of 64, read through the sums' term_c_off; not with NO_FUSE1X1_MERGE);
      BN folding; the stride-2 256-channel K split of transition1.1 (TF32 and bf16: two 128-channel parts chained through
      res, bias on part 0, ReLU on the last part); the fused head-in conv (head order 3, 1, 2, in_c_off / res_c_off 64 s,
      the coord channels folded into a res_broadcast bias map, pow_channel 0 on the cam head, params_maps written at
      out_c_off 0 and 3).  Six distinct records: fp32, and TF32 = bf16, per switch.
  ROMP ResNet-50 {fp32, tf32, bf16} x {default, B200ROMP_NO_S2_KSPLIT=1, B200ROMP_S2_KSPLIT_C=64}: backbone_out,
      center_maps, params_maps.  Rewrites: the stem with the normalisation folded into w / (255 std) and a broadcast bias
      map of the zero-padded normalised image; MaxPool2d(3, 2, 1); the stride-2 256-channel K split of layer3.0 conv2
      (TF32 and bf16 only; parts chained through res, bias on part 0, ReLU on the last part; 128 channels per part, 64 with
      S2_KSPLIT_C=64, none with NO_S2_KSPLIT in bf16), asserted to split that conv and nothing else; BN folded into the
      three ConvTranspose2d(4, 2, 1); the fused head-in conv on 64 + 2 channels.  Three distinct records: no split,
      128-channel parts, 64-channel parts.
  BEV {fp32, tf32, bf16}: G1 maps_fv, fv_feats, img_feats (the first 16 channels; in bf16 channels 16..31 must be exactly
      0); G2 bv_out, fed with the bird's-eye input the oracle gives its bv_out_layers.  Rewrites: the HRNet backbone as
      above; head_block with its biased 1x1 residual conv; bv_pre_layers zero-padded to 32 channels (bf16 only); the G2
      Conv1d stack (ksize code 13).  Two distinct records: fp32 = tf32, bf16.
Negative controls mutate a record (or the builder) and must be rejected: the [W3 | Wd] halves swapped, one merged-1x1
term_c_off shifted by one channel, the K-split bias on parts 0 and 1, the last K-split part's ReLU dropped, the cam and
params head slices swapped, the coord channels of the head bias map transposed, the stem bias map computed from
zero-padded raw pixels (the interior value everywhere), a nonzero weight row in a BEV padding channel, the G2 Conv1d taps
reversed.  Moving the K-split bias from part 0 to part 1 is exact algebra (no ReLU between the parts): it must be
accepted.

test_bf16_rounding records every bf16 graph a second time with the real round_bf16: every conv weight array must be the
round-to-nearest-even bf16 (computed here on the bits) of the same array in the unrounded record, the ConvTranspose2d
weights (fp32 multiplies on the CUDA cores) and every bias and constant tensor unchanged, zeros (the padding) still zero.

test_fake_record_matches_library (GPU): for every graph of the matrix, the FakeLib record equals, call for call, the
record the Recorder makes through the real library: the same descriptors, weight and constant bytes, lanes and finalize
batch.  So what is interpreted here is what ships.

Runtime: without a GPU the file takes 74 s on an 8-core x86 CPU (the float64 interpreter: 2.5 - 4 s per HRNet or BEV
G1 record, 1.2 - 2 s per ResNet-50 record; 12 distinct records and 10 negative-control interpretations).  That is short
enough that the float64 math always runs on the CPU.  On a machine with one H100 80GB HBM3 at a 700 W power limit the
whole file, the 21 recording-equality builds included, takes 98 s.
"""
import ctypes as C
import hashlib
import time

import numpy as np
import pytest
import torch

from oracle import bev_oracle as B
from oracle import romp_oracle as R
from romp_b200 import _lib, graph, synth
from romp_b200._lib import U8
from tests.net_graphs import aliasing_violations
from tests.test_gpu_graph_ops import (Recorder, conv_linear, excess, maxpool_ref, normalise_input, pow_f32_11, record,
                                      sum_terms)

BOUND = 2.0 ** -18          # |v - ref| <= BOUND * A (module docstring)
REJECT = 100                # a negative control's worst |v - ref| / (BOUND A) must exceed this
PRECISIONS = ("fp32", "tf32", "bf16")
ROMP_SWITCHES = {"default": {}, "NO_SKIP_CONCAT": {"B200ROMP_NO_SKIP_CONCAT": "1"},
                 "NO_FUSE1X1_MERGE": {"B200ROMP_NO_FUSE1X1_MERGE": "1"}}
R50_SWITCHES = {"default": {}, "NO_S2_KSPLIT": {"B200ROMP_NO_S2_KSPLIT": "1"}, "S2_KSPLIT_C=64": {"B200ROMP_S2_KSPLIT_C": "64"}}
SWITCH_VARS = ("B200ROMP_NO_SKIP_CONCAT", "B200ROMP_NO_FUSE1X1_MERGE", "B200ROMP_NO_S2_KSPLIT", "B200ROMP_S2_KSPLIT_C")
MAX_BATCH = 2
FRAME_SEED = 5


# ---------------------------------------------------------------------------------------------------------------------
# recording without the library
# ---------------------------------------------------------------------------------------------------------------------
class _Ids:
    """the graph-building calls of libb200romp without a device: tensor and op ids numbered as the library numbers them
    (net.cu: one counter per net for tensors, const tensors included, one for ops)"""

    def __init__(self):
        self.n_tensors, self.n_ops = {}, {}

    def b200romp_net_create(self, dev):
        net = len(self.n_tensors) + 1
        self.n_tensors[net], self.n_ops[net] = 0, 0
        return net

    def _tensor(self, net):
        self.n_tensors[net] += 1
        return self.n_tensors[net] - 1

    def _op(self, net):
        self.n_ops[net] += 1
        return self.n_ops[net] - 1

    def b200romp_net_add_tensor(self, net, H, W, Cc, dt, nchw, ext):
        return self._tensor(net)

    def b200romp_net_add_const_tensor(self, net, H, W, Cc, dt, ptr):
        return self._tensor(net)

    def b200romp_net_add_conv(self, net, dref, wp, bp):
        return self._op(net)

    def b200romp_net_add_sum(self, net, sref):
        return self._op(net)

    def b200romp_net_add_maxpool(self, net, i, o):
        return self._op(net)

    def b200romp_net_set_lane(self, net, op, lane):
        assert 0 <= op < self.n_ops[net]
        return 0

    def b200romp_net_finalize(self, net, max_batch):
        return 0

    def b200romp_last_error(self):
        return b""


class FakeLib(Recorder):
    """stands in for _lib.load() while a builder runs: the Recorder's copies of every descriptor, weight, bias and constant
    tensor, over _Ids instead of the library"""

    def __init__(self):
        super().__init__(_Ids())


def fake_record(monkeypatch, build, env=None, bf16_rounding=False):
    """run build() against FakeLib with the switch variables `env` set -> (build's result, [record per net]).  Without
    bf16_rounding, graph.round_bf16 is the identity: bf16 graphs keep their fp32 folded weights."""
    fake = FakeLib()
    with monkeypatch.context() as m:
        for k in SWITCH_VARS:
            m.delenv(k, raising=False)
        for k, v in (env or {}).items():
            m.setenv(k, v)
        m.setattr(_lib, "load", lambda: fake)
        if not bf16_rounding:
            m.setattr(graph, "round_bf16", lambda a: a)
        out = build()
    return out, fake.nets


def builder(kind, sd, precision):
    build = {"romp": graph.build_romp, "resnet50": graph.build_romp_resnet50, "bev": graph.build_bev}[kind]
    return lambda: build(sd, 0, precision, U8, MAX_BATCH)


def semantic_key(r):
    """what the interpreter reads of a record: ops, descriptors without the engine, tensor shapes without the dtype,
    weight, bias and constant bytes (lanes and dtypes do not change what is computed)"""
    h = hashlib.sha1()
    for kind, rid, args in r["calls"]:
        if kind == "tensor":
            H, W, Cc, dt, nchw, ext = args
            h.update(repr((kind, rid, H, W, Cc, nchw, ext)).encode())
        elif kind == "const":
            h.update(repr((kind, rid) + args[:3]).encode())
            h.update(args[4].tobytes())
        elif kind == "conv":
            d, w, b = args
            h.update(repr((kind, rid) + tuple(getattr(d, f) for f, _ in d._fields_ if f != "engine")).encode())
            h.update(w.tobytes())
            h.update(b"-" if b is None else b.tobytes())
        elif kind == "sum":
            h.update(repr((kind, rid)).encode() + C.string_at(C.byref(args[0]), C.sizeof(args[0])))
        elif kind == "maxpool":
            h.update(repr((kind, rid, args)).encode())
    return h.hexdigest()


# ---------------------------------------------------------------------------------------------------------------------
# the float64 interpreter
# ---------------------------------------------------------------------------------------------------------------------
def _reads(kind, args):
    if kind == "conv":
        d = args[0]
        return [d.in_] + ([d.res] if d.res >= 0 else [])
    if kind == "sum":
        s = args[0]
        return [s.base] + [s.term[k] for k in range(s.n_terms)]
    return [args[0]]


def conv_weights(d, w, b):
    """recorded weight and bias arrays -> float64 tensors in the layout of ksize code d.ksize"""
    shape = ((d.cout, d.cin, 3) if d.ksize == 13 else (d.cin, d.cout, 4, 4) if d.ksize == 42
             else (d.cout, d.cin, d.ksize, d.ksize))
    return torch.from_numpy(w.reshape(shape)).double(), None if b is None else torch.from_numpy(b).double()


def interpret(r, inputs, keep):
    """run record r in float64 on one frame.  inputs: {tensor id: NHWC tensor [1, H, W, C]} (NCHW tensors are held
    NHWC too); keep: the tensor ids to return.  -> ({id: v}, {id: A}, longest conv path to each kept tensor).
    A is the magnitude an op summed its output from, the op applied to |inputs|, |W|, |b| plus |res| (as in conv_bound
    and sum_bound); a maxpool passes on the largest A of its window."""
    info = r["tensors"]
    ops = [(kind, args) for kind, _, args in r["calls"] if kind in ("conv", "sum", "maxpool")]
    last = {}
    for i, (kind, args) in enumerate(ops):
        for t in _reads(kind, args):
            last[t] = i
    V = {t: x.double() for t, x in inputs.items()}
    A = {}
    depth = {t: 0 for t in info}
    for kind, rid, args in r["calls"]:
        if kind == "const":
            H, W, Cc, _, data = args
            V[rid] = torch.from_numpy(data).double().view(1, H, W, Cc)

    def out(t):
        if t not in V:
            s = info[t]
            V[t] = torch.zeros(1, s["H"], s["W"], s["C"], dtype=torch.float64)
            A[t] = torch.zeros_like(V[t])
        return V[t], A[t]

    for i, (kind, args) in enumerate(ops):
        if kind == "conv":
            d, w, b = args
            wt, bt = conv_weights(d, w, b)
            x = V[d.in_][..., d.in_c_off:d.in_c_off + d.cin]
            if d.input_norm:
                x = normalise_input(x)
            kw = dict(stride=d.stride, up=d.upsample, transpose=d.ksize == 42)
            z = conv_linear(x, wt, bt, **kw)
            a = conv_linear(x.abs(), wt.abs(), None if bt is None else bt.abs(), **kw)
            if d.res >= 0:
                res = V[d.res][..., d.res_c_off:d.res_c_off + d.cout]
                z = z + res
                a = a + res.abs()
            if d.relu:
                z = z.clamp_min(0)
            if d.pow_channel >= 0:
                c = d.pow_channel
                z[..., c] = pow_f32_11(z[..., c])
                a[..., c] = z[..., c] * a[..., c]
            vo, ao = out(d.out)
            vo[..., d.out_c_off:d.out_c_off + d.cout] = z
            ao[..., d.out_c_off:d.out_c_off + d.cout] = a
            depth[d.out] = max(depth[d.out], 1 + max(depth[t] for t in _reads(kind, args)))
        elif kind == "sum":
            s = args[0]
            Cc = info[s.out]["C"]
            ts = [(s.term[k], s.term_c_off[k]) for k in range(s.n_terms)]
            ups = [s.up[k] for k in range(s.n_terms)]
            z = sum_terms(V[s.base], [V[t][..., o:o + Cc] for t, o in ts], ups)
            vo, ao = out(s.out)
            vo[:] = z.clamp_min(0) if s.relu else z
            ao[:] = sum_terms(V[s.base].abs(), [V[t][..., o:o + Cc].abs() for t, o in ts], ups)
            depth[s.out] = max(depth[t] for t in _reads(kind, args))
        else:
            src, dst = args
            vo, ao = out(dst)
            vo[:], ao[:] = maxpool_ref(V[src]), maxpool_ref(A[src])
            depth[dst] = depth[src]
        for t in _reads(kind, args):
            if last[t] == i and t not in keep:
                V.pop(t, None)
                A.pop(t, None)
    return {t: V[t] for t in keep}, {t: A[t] for t in keep}, {t: depth[t] for t in keep}


def ratio(v, ref, a):
    """worst |v - ref| / (BOUND A) and the number of elements over the bound"""
    return excess(v, ref, BOUND * a)


# ---------------------------------------------------------------------------------------------------------------------
# the oracle in float64
# ---------------------------------------------------------------------------------------------------------------------
def _sd64(sd):
    return {k: torch.from_numpy(np.asarray(v)).double() if np.asarray(v).dtype.kind == "f" else torch.from_numpy(np.asarray(v))
            for k, v in sd.items()}


def _nhwc(t):
    return t.permute(0, 2, 3, 1)


@pytest.fixture(scope="module")
def frame():
    return torch.from_numpy(synth.synthetic_frames(1, seed=FRAME_SEED))


@pytest.fixture(scope="module")
def romp_sd():
    return synth.romp_state_dict(0)


@pytest.fixture(scope="module")
def resnet50_sd():
    return synth.resnet50_state_dict(0)


@pytest.fixture(scope="module")
def bev_sd():
    return synth.bev_state_dict(0)


@pytest.fixture(scope="module")
def romp_ref(romp_sd, frame):
    sd = _sd64(romp_sd)
    x = frame.double()
    with torch.no_grad():
        center, params = R.romp_maps(sd, x, torch.float64)
        feat = R.hrnet32_forward(sd, x)
    return dict(backbone_out=_nhwc(feat), center_maps=_nhwc(center), params_maps=_nhwc(params))


@pytest.fixture(scope="module")
def resnet50_ref(resnet50_sd, frame):
    sd = _sd64(resnet50_sd)
    x = frame.double()
    with torch.no_grad():
        center, params = R.romp_resnet50_maps(sd, x, torch.float64)
        feat = R.resnet50_forward(sd, x)
    return dict(backbone_out=_nhwc(feat), center_maps=_nhwc(center), params_maps=_nhwc(params))


@pytest.fixture(scope="module")
def bev_ref(bev_sd, frame):
    sd = _sd64(bev_sd)
    with torch.no_grad():
        feat = R.hrnet32_forward(sd, frame.double())
        maps_fv, img_feats = B.fv_maps(sd, feat)
        fv = B.head_block(sd, "param_head.0.0.", feat)
        summon = B.bv_input(maps_fv, img_feats)
        bv = B.bv_out(sd, summon)
    # G2's tensors: bv_in [1, 128 (W), 2560 (C)], bv_out [1, 128 (W), 128 (C)]
    return dict(maps_fv=_nhwc(maps_fv), fv_feats=_nhwc(fv), img_feats=_nhwc(img_feats),
                bv_in=summon.transpose(1, 2)[:, None], bv_out=bv.transpose(1, 2)[:, None])


# ---------------------------------------------------------------------------------------------------------------------
# one graph against the oracle
# ---------------------------------------------------------------------------------------------------------------------
_RESULTS = {}      # semantic key -> {output: (worst ratio, elements over, longest path)}


def compare(r, inputs, outputs, ref, pad_zero=()):
    """interpret record r and compare `outputs` {name: tensor id} with ref {name: NHWC float64}; a reference with fewer
    channels than the tensor covers its first channels, and the rest must be exactly 0 (pad_zero names the outputs where
    that is expected).  -> {name: (worst ratio, elements over the bound, longest path)}"""
    v, a, depth = interpret(r, inputs, set(outputs.values()))
    res = {}
    for name, t in outputs.items():
        c = ref[name].shape[-1]
        res[name] = ratio(v[t][..., :c], ref[name], a[t][..., :c]) + (depth[t],)
        if v[t].shape[-1] > c:
            assert name in pad_zero, f"{name}: {v[t].shape[-1]} channels, the model has {c}"
            rest = v[t][..., c:]
            pad = excess(rest, torch.zeros_like(rest), BOUND * a[t][..., c:])
            res[name + f"[{c}:]"] = (pad[0] if rest.any() else 0.0, int((rest != 0).sum()), depth[t])
    return res


def cached_compare(r, inputs, outputs, ref, label, pad_zero=()):
    key = semantic_key(r)
    seen = key in _RESULTS
    if not seen:
        t0 = time.time()
        _RESULTS[key] = (compare(r, inputs, outputs, ref, pad_zero), label, time.time() - t0)
    res, first, dt = _RESULTS[key]
    how = f"the record of {first}" if seen else f"interpreted in {dt:.1f} s"
    for name, (worst, over, depth) in res.items():
        print(f"   {label} {name}: worst |v - ref| / (2^-18 A) {worst:.3g}, {over} elements over, longest conv path "
              f"{depth}  ({how})", flush=True)
    return res


def assert_within(res, label):
    bad = {k: v for k, v in res.items() if v[1]}
    assert not bad, f"{label}: elements over the bound: {bad}"


def ksplit_parts(r):
    """the K-split stride-2 convs of record r: [[part convs] per split conv]; a part is a stride-2 3x3 conv reading a
    channel slice narrower than its input tensor, and the parts of one conv are chained through res"""
    info = r["tensors"]
    convs = [a[0] for k, _, a in r["calls"] if k == "conv"]
    splits = []
    for d in convs:
        if d.ksize == 3 and d.stride == 2 and d.cin < info[d.in_]["C"] and d.in_c_off == 0 and d.res < 0:
            chain = [d]
            while True:
                nxt = [e for e in convs if e.res == chain[-1].out and e.in_ == d.in_]
                if not nxt:
                    break
                chain.append(nxt[0])
            splits.append(chain)
    return splits


def check_split(r, n, in_hw, out_hwc):
    """the one stride-2 3x3 conv of 256 input channels in record r (input at in_hw, output out_hwc) is split into n parts
    (0: not split): consecutive 256 / n channel slices, chained through res, bias on part 0, ReLU on the last part"""
    info = r["tensors"]
    splits = ksplit_parts(r)
    whole = [a[0] for k, _, a in r["calls"] if k == "conv" and a[0].ksize == 3 and a[0].stride == 2 and a[0].cin == 256]
    if not n:
        assert not splits and len(whole) == 1
        parts = whole
    else:
        assert len(splits) == 1 and not whole, splits
        parts = splits[0]
        assert len(parts) == n and all(p.cin == 256 // n for p in parts)
        assert [p.in_c_off for p in parts] == [i * 256 // n for i in range(n)]
        assert [p.relu for p in parts] == [0] * (n - 1) + [1]
        assert [p.res for p in parts[1:]] == [p.out for p in parts[:-1]]
        biased = [a[2] is not None for k, _, a in r["calls"] if k == "conv" and any(a[0] is p for p in parts)]
        assert biased == [True] + [False] * (n - 1)
    t, o = info[parts[0].in_], info[parts[-1].out]
    assert (t["H"], t["W"], t["C"]) == in_hw + (256,) and (o["H"], o["W"], o["C"]) == out_hwc


# ---------------------------------------------------------------------------------------------------------------------
# the matrix
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("switch", list(ROMP_SWITCHES))
@pytest.mark.parametrize("precision", PRECISIONS)
def test_romp_graph_semantics(monkeypatch, romp_sd, romp_ref, frame, precision, switch):
    built, (r,) = fake_record(monkeypatch, builder("romp", romp_sd, precision), ROMP_SWITCHES[switch])
    nb, io = built
    outputs = dict(backbone_out=nb.names["backbone_out"], center_maps=io["center_maps"], params_maps=io["params_maps"])
    convs = [a[0] for k, _, a in r["calls"] if k == "conv"]
    concat = [d for d in convs if d.ksize == 1 and d.cin == 128 and d.cout == 256]
    assert len(concat) == (0 if switch == "NO_SKIP_CONCAT" else 1)
    merged = [a[0] for k, _, a in r["calls"] if k == "sum" and any(a[0].term_c_off[j] for j in range(a[0].n_terms))]
    assert (len(merged) == 0) == (switch == "NO_FUSE1X1_MERGE")
    # transition1.1: 256 channels at 128x128 -> 64 at 64x64, split on TF32 and bf16
    check_split(r, 0 if precision == "fp32" else 2, (128, 128), (64, 64, 64))
    res = cached_compare(r, {io["frames"]: frame}, outputs, romp_ref, f"ROMP {precision} {switch}")
    assert_within(res, f"ROMP {precision} {switch}")


# parts of layer3.0 conv2 (256 channels, stride 2): no split on the SIMT engine, 128 channels per part on TF32, the
# switches act in bf16 only
KSPLIT_PARTS = {("fp32", s): 0 for s in R50_SWITCHES}
KSPLIT_PARTS.update({("tf32", s): 2 for s in R50_SWITCHES})
KSPLIT_PARTS.update({("bf16", "default"): 2, ("bf16", "NO_S2_KSPLIT"): 0, ("bf16", "S2_KSPLIT_C=64"): 4})


@pytest.mark.parametrize("switch", list(R50_SWITCHES))
@pytest.mark.parametrize("precision", PRECISIONS)
def test_resnet50_graph_semantics(monkeypatch, resnet50_sd, resnet50_ref, frame, precision, switch):
    built, (r,) = fake_record(monkeypatch, builder("resnet50", resnet50_sd, precision), R50_SWITCHES[switch])
    nb, io = built
    outputs = dict(backbone_out=nb.names["backbone_out"], center_maps=io["center_maps"], params_maps=io["params_maps"])
    # layer3.0 conv2: 256 channels at 64x64 -> 256 at 32x32
    check_split(r, KSPLIT_PARTS[(precision, switch)], (64, 64), (32, 32, 256))
    res = cached_compare(r, {io["frames"]: frame}, outputs, resnet50_ref, f"ROMP ResNet-50 {precision} {switch}")
    assert_within(res, f"ROMP ResNet-50 {precision} {switch}")


@pytest.mark.parametrize("precision", PRECISIONS)
def test_bev_graph_semantics(monkeypatch, bev_sd, bev_ref, frame, precision):
    (g1, io1, g2, io2), (r1, r2) = fake_record(monkeypatch, builder("bev", bev_sd, precision))
    assert r1["tensors"][io1["img_feats"]]["C"] == (32 if precision == "bf16" else 16)
    outs1 = dict(maps_fv=io1["maps_fv"], fv_feats=io1["fv_feats"], img_feats=io1["img_feats"])
    res = cached_compare(r1, {io1["frames"]: frame}, outs1, bev_ref, f"BEV {precision} G1", pad_zero=("img_feats",))
    if precision == "bf16":
        assert res["img_feats[16:]"][1] == 0, "img_feats channels 16..31 are not exactly 0"
    assert_within(res, f"BEV {precision} G1")
    res = cached_compare(r2, {io2["bv_in"]: bev_ref["bv_in"]}, dict(bv_out=io2["bv_out"]), bev_ref, f"BEV {precision} G2")
    assert_within(res, f"BEV {precision} G2")


# ---------------------------------------------------------------------------------------------------------------------
# the bf16 weight rounding
# ---------------------------------------------------------------------------------------------------------------------
def rne_bf16(a):
    """fp32 -> bf16 round to nearest, ties to even, on the bits; the result in fp32"""
    u = np.ascontiguousarray(a, np.float32).view(np.uint32).astype(np.uint64)
    return ((u + 0x7FFF + ((u >> 16) & 1)) & 0xFFFF0000).astype(np.uint32).view(np.float32)


def _same_desc(a, b):
    return C.string_at(C.byref(a), C.sizeof(a)) == C.string_at(C.byref(b), C.sizeof(b))


BF16_GRAPHS = ([("romp", s, e) for s, e in ROMP_SWITCHES.items()] + [("resnet50", s, e) for s, e in R50_SWITCHES.items()]
               + [("bev", "default", {})])


@pytest.mark.parametrize("kind,switch,env", BF16_GRAPHS, ids=[f"{k}-{s}" for k, s, _ in BF16_GRAPHS])
def test_bf16_rounding(monkeypatch, romp_sd, resnet50_sd, bev_sd, kind, switch, env):
    sd = dict(romp=romp_sd, resnet50=resnet50_sd, bev=bev_sd)[kind]
    _, plain = fake_record(monkeypatch, builder(kind, sd, "bf16"), env)
    _, rounded = fake_record(monkeypatch, builder(kind, sd, "bf16"), env, bf16_rounding=True)
    n_conv = n_rounded = 0
    for rp, rr in zip(plain, rounded, strict=True):
        assert rp["max_batch"] == rr["max_batch"]
        for (kp, ip, ap), (kr, ir, ar) in zip(rp["calls"], rr["calls"], strict=True):
            assert (kp, ip) == (kr, ir)
            if kp == "conv":
                (dp, wp, bp), (dr, wr, br) = ap, ar
                assert _same_desc(dp, dr)
                n_conv += 1
                if dp.ksize == 42:      # ConvTranspose2d(4, 2, 1): fp32 weights, the CUDA cores multiply them
                    assert wr.tobytes() == wp.tobytes()
                else:
                    assert wr.tobytes() == rne_bf16(wp).tobytes(), f"conv {ip}: weights are not the RNE bf16 of the fold"
                    n_rounded += int((wr != wp).any())
                assert (wr[wp == 0] == 0).all(), "a zero weight (padding) became nonzero"
                assert (bp is None) == (br is None) and (bp is None or bp.tobytes() == br.tobytes()), f"conv {ip}: bias"
            elif kp == "const":
                assert ap[:4] == ar[:4] and ap[4].tobytes() == ar[4].tobytes(), f"const tensor {ip} changed"
            elif kp == "sum":
                assert _same_desc(ap[0], ar[0])
            else:
                assert ap == ar
    print(f"   bf16 {kind} {switch}: {n_conv} convs, {n_rounded} with weights changed by the rounding")
    assert n_rounded > 0.9 * n_conv - 3


# ---------------------------------------------------------------------------------------------------------------------
# negative controls
# ---------------------------------------------------------------------------------------------------------------------
def mutated(r, i, args):
    """a copy of record r with call i's arguments replaced"""
    calls = list(r["calls"])
    kind, rid, _ = calls[i]
    calls[i] = (kind, rid, args)
    return dict(r, calls=calls)


def copy_desc(d, **kw):
    e = type(d)()
    C.memmove(C.byref(e), C.byref(d), C.sizeof(d))
    for k, v in kw.items():
        setattr(e, k, v)
    return e


def conv_calls(r, pred):
    return [i for i, (k, _, a) in enumerate(r["calls"]) if k == "conv" and pred(a[0])]


def rejected(what, r, inputs, outputs, ref, pad_zero=()):
    res = compare(r, inputs, outputs, ref, pad_zero)
    worst = max(v[0] for v in res.values())
    print(f"   negative control {what}: worst |v - ref| / (2^-18 A) {worst:.3g} -> "
          f"{'rejected' if worst > REJECT else 'NOT rejected'}", flush=True)
    assert worst > REJECT, f"negative control not rejected: {what} ({res})"


def test_negative_controls_romp(monkeypatch, romp_sd, romp_ref, frame):
    (nb, io), (r,) = fake_record(monkeypatch, builder("romp", romp_sd, "fp32"))
    outputs = dict(backbone_out=nb.names["backbone_out"], center_maps=io["center_maps"], params_maps=io["params_maps"])
    inputs = {io["frames"]: frame}

    (i,) = conv_calls(r, lambda d: d.ksize == 1 and d.cin == 128 and d.cout == 256)
    d, w, b = r["calls"][i][2]
    w4 = w.reshape(256, 128)
    rejected("[W3 | Wd] halves swapped", mutated(r, i, (d, np.concatenate([w4[:, 64:], w4[:, :64]], 1).ravel(), b)),
             inputs, outputs, romp_ref)

    i, k = next((i, k) for i, (kind, _, a) in enumerate(r["calls"]) if kind == "sum"
                for k in range(a[0].n_terms) if a[0].term_c_off[k] > 0)
    s = copy_desc(r["calls"][i][2][0])
    s.term_c_off[k] -= 1
    rejected("merged 1x1 term_c_off shifted by one channel", mutated(r, i, (s,)), inputs, outputs, romp_ref)

    hin = nb.names["head_in"]
    r2 = r
    for i in conv_calls(r, lambda d: d.in_ == hin or d.res == hin):
        d, w, b = r["calls"][i][2]
        swap = {0: 64, 64: 0, 128: 128}
        d = copy_desc(d, in_c_off=swap[d.in_c_off]) if d.in_ == hin else copy_desc(d, res_c_off=swap[d.res_c_off])
        r2 = mutated(r2, i, (d, w, b))
    rejected("cam and params head slices swapped", r2, inputs, outputs, romp_ref)

    coord = graph.coord_maps
    monkeypatch.setattr(graph, "coord_maps", lambda size=128: coord(size).flip(1).contiguous())
    (nb3, io3), (r3,) = fake_record(monkeypatch, builder("romp", romp_sd, "fp32"))
    monkeypatch.setattr(graph, "coord_maps", coord)
    rejected("coord channels of the head bias map transposed", r3, inputs, outputs, romp_ref)


def test_negative_controls_resnet50(monkeypatch, resnet50_sd, resnet50_ref, frame):
    (nb, io), (r,) = fake_record(monkeypatch, builder("resnet50", resnet50_sd, "tf32"))
    outputs = dict(backbone_out=nb.names["backbone_out"], center_maps=io["center_maps"], params_maps=io["params_maps"])
    inputs = {io["frames"]: frame}
    (parts,) = ksplit_parts(r)
    i0, i1 = (conv_calls(r, lambda d, p=p: d.out == p.out and d.in_c_off == p.in_c_off)[0] for p in parts[:2])
    (d0, w0, b0), (d1, w1, b1) = r["calls"][i0][2], r["calls"][i1][2]
    assert b0 is not None and b1 is None
    # no ReLU between the parts: the bias may sit on any one part (exact algebra, accepted); on two it counts twice
    res = compare(mutated(mutated(r, i0, (d0, w0, None)), i1, (d1, w1, b0)), inputs, outputs, resnet50_ref)
    worst = max(v[0] for v in res.values())
    print(f"   equivalent rewrite, the K-split bias on part 1 instead of part 0: worst |v - ref| / (2^-18 A) {worst:.3g}"
          f" -> accepted")
    assert worst < 1
    rejected("K-split bias on parts 0 and 1", mutated(r, i1, (d1, w1, b0)), inputs, outputs, resnet50_ref)
    il = conv_calls(r, lambda d: d.out == parts[-1].out and d.in_c_off == parts[-1].in_c_off)[0]
    dl, wl, bl = r["calls"][il][2]
    rejected("last K-split part without its ReLU", mutated(r, il, (copy_desc(dl, relu=0), wl, bl)), inputs, outputs,
             resnet50_ref)

    (i,) = [i for i, (k, rid, a) in enumerate(r["calls"]) if k == "const" and rid == nb.names["stem_bias_map"]]
    H, W, Cc, dt, data = r["calls"][i][2]
    m = data.reshape(H, W, Cc)
    interior = np.broadcast_to(m[H // 2, W // 2], m.shape).ravel().copy()
    assert not np.array_equal(interior, data)
    rejected("stem bias map of zero-padded raw pixels", mutated(r, i, (H, W, Cc, dt, interior)), inputs, outputs,
             resnet50_ref)


def test_negative_controls_bev(monkeypatch, bev_sd, bev_ref, frame):
    (g1, io1, g2, io2), (r1, r2) = fake_record(monkeypatch, builder("bev", bev_sd, "bf16"))
    (i,) = conv_calls(r1, lambda d: d.out == io1["img_feats"])
    d, w, b = r1["calls"][i][2]
    w2 = w.reshape(d.cout, d.cin).copy()
    assert not w2[16:].any()
    w2[20] = w2[0]
    rejected("nonzero weights in a padding channel of bv_pre_layers", mutated(r1, i, (d, w2.ravel(), b)),
             {io1["frames"]: frame}, dict(img_feats=io1["img_feats"]), bev_ref, pad_zero=("img_feats",))

    i = conv_calls(r2, lambda d: d.ksize == 13)[0]
    d, w, b = r2["calls"][i][2]
    rev = np.ascontiguousarray(w.reshape(d.cout, d.cin, 3)[..., ::-1]).ravel()
    rejected("G2 Conv1d taps reversed", mutated(r2, i, (d, rev, b)), {io2["bv_in"]: bev_ref["bv_in"]},
             dict(bv_out=io2["bv_out"]), bev_ref)


# ---------------------------------------------------------------------------------------------------------------------
# the CPU record is the record of what ships
# ---------------------------------------------------------------------------------------------------------------------
def records_equal(a, b, label):
    assert len(a) == len(b), label
    for ra, rb in zip(a, b):
        assert ra["max_batch"] == rb["max_batch"], label
        assert len(ra["calls"]) == len(rb["calls"]), label
        for n, ((ka, ia, aa), (kb, ib, ab)) in enumerate(zip(ra["calls"], rb["calls"])):
            where = f"{label}: call {n} ({ka} {ia})"
            assert (ka, ia) == (kb, ib), where
            if ka == "conv":
                assert _same_desc(aa[0], ab[0]), where
                assert aa[1].tobytes() == ab[1].tobytes(), where + ": weights"
                assert (aa[2] is None) == (ab[2] is None) and (aa[2] is None or aa[2].tobytes() == ab[2].tobytes()), where
            elif ka == "sum":
                assert _same_desc(aa[0], ab[0]), where
            elif ka == "const":
                assert aa[:4] == ab[:4] and aa[4].tobytes() == ab[4].tobytes(), where
            else:
                assert aa == ab, where


MATRIX = ([("romp", p, s, e) for p in PRECISIONS for s, e in ROMP_SWITCHES.items()]
          + [("resnet50", p, s, e) for p in PRECISIONS for s, e in R50_SWITCHES.items()]
          + [("bev", p, "default", {}) for p in PRECISIONS])


@pytest.mark.gpu
@pytest.mark.parametrize("kind,precision,switch,env", MATRIX, ids=[f"{k}-{p}-{s}" for k, p, s, _ in MATRIX])
def test_fake_record_matches_library(monkeypatch, romp_sd, resnet50_sd, bev_sd, kind, precision, switch, env):
    sd = dict(romp=romp_sd, resnet50=resnet50_sd, bev=bev_sd)[kind]
    _, fake = fake_record(monkeypatch, builder(kind, sd, precision), env, bf16_rounding=True)
    with monkeypatch.context() as m:
        for k in SWITCH_VARS:
            m.delenv(k, raising=False)
        for k, v in env.items():
            m.setenv(k, v)
        built, real = record(m, builder(kind, sd, precision))
    records_equal(fake, real, f"{kind} {precision} {switch}")
    for nb in built if kind == "bev" else built[:1]:
        if isinstance(nb, graph.NetBuilder):
            nb.lib.b200romp_net_destroy(nb.net)


@pytest.mark.parametrize("kind,precision,switch,env", MATRIX, ids=[f"{k}-{p}-{s}" for k, p, s, _ in MATRIX])
def test_builder_graphs_keep_aliasing_rule(monkeypatch, romp_sd, resnet50_sd, bev_sd, kind, precision, switch, env):
    """no graph the builder emits has an op whose read slice of its output tensor overlaps the output slice without
    being it (include/b200romp.h): the check add_conv / add_maxpool make and the no-fusion rule for in-place chains
    leave every shipped plan as it was"""
    sd = dict(romp=romp_sd, resnet50=resnet50_sd, bev=bev_sd)[kind]
    _, recs = fake_record(monkeypatch, builder(kind, sd, precision), env)
    for r in recs:
        assert not aliasing_violations(r), f"{kind} {precision} {switch}: {aliasing_violations(r)}"
        chains = [d for k, _, a in r["calls"] if k == "conv" for d in [a[0]] if d.res >= 0 and d.res == d.out]
        assert not chains, f"{kind} {precision} {switch}: in-place residual convs {[(d.in_, d.out) for d in chains]}"
