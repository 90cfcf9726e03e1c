"""The diagnostic paths behind the environment switches (INTEGRATION.md, "Environment switches of `libb200romp.so`"),
checked against float64 like the production path, and shown to have run.

Graph-builder switches (B200ROMP_NO_SKIP_CONCAT, B200ROMP_NO_FUSE1X1_MERGE, B200ROMP_NO_S2_KSPLIT,
B200ROMP_S2_KSPLIT_C=64) are read by graph.py while a graph is built, so they are set in this process with monkeypatch:
every op of the switched ROMP HRNet bf16 (batch 64), ROMP ResNet-50 bf16 (batch 64) and BEV G1 bf16 (batch 34) graph
is checked in place by test_gpu_graph_ops.verify_graph (the batches of that file: some CTA of every persistent op runs a
third tile, or the op is rerun alone at a batch that gives it one), and the describe() plan must differ from the
default build as the switch says.  A switch whose graph has the default plan fails.

Library switches are latched once per process, into function-local statics, at the first launch that reads them: setting
them after the library has run does nothing.  Each one therefore runs in a child pytest process of this file that has the
variable in its environment from the start; test_child_* skip unless B200ROMP_SWITCH_CHILD names them, so a normal run
collects them as skipped, and the children run one after another.  What a child checks, and how it shows its path ran:
  SUM_SIMPLE, SUM_RING (and SUM_RING with NO_FUSE1X1_MERGE, whose sums read whole tensors, the only terms the ring kernel
      takes): the standalone shapes of test_gpu_fuse_sum against a float64 sum and bit for bit against the fp32 sum in the
      kernels' order, and every op of the ROMP bf16 (batch 64) and TF32 (batch 34) graphs in place.  Each sum op's
      describe() line names the kernel it takes ([fuse-sum ring|pipe|simple]); every sum must take the expected one.
  TC_NO_FOLD: the 32->32 cases of test_gpu_conv_tc and every op of the ROMP bf16 graph; describe() shows no pixel-pair
      fold and no fused 32-channel block.
  NO_PDL: the outputs of the ROMP bf16 and TF32 graphs and of both BEV bf16 graphs are bit-identical to the default run on
      the same seeded inputs (written by the parent, which runs the default path).  A difference means a kernel reads its
      predecessor's output before its pdl_wait.  There is no plan to show: the child asserts the variable came with the
      process, before the library was loaded.
  BEV_CENTER3D_2PASS: test_gpu_bev_detect_fp64.check_center3d on the model state and on the crafted inputs (fp32 and bf16,
      batches 1, 3 and 32), with the per-voxel float64 bound of the fused kernel.  The two-pass kernel writes its
      intermediate into `tmp`, which the fused kernel never touches: `tmp` is filled with NaN first and must come back
      finite.

Measured on one H100 80GB HBM3 at a 700 W power limit: the file takes 3 min 10 s - 3 min 25 s, about 4.5 times
test_gpu_graph_ops.py (45 s).  The six children take 15 - 27 s each (2 min 20 s together), mostly Python start-up, library
load and graph builds before their own checks; the in-process graph-builder tests take about 55 s.  Peak device memory is that of the ROMP bf16 graph at
batch 64 with every tensor kept: 12 - 14 GiB.
"""
import ctypes as C
import os
import re
import subprocess
import sys
import time
from collections import Counter

import numpy as np
import pytest
import torch

from romp_b200 import _lib, graph, synth
from romp_b200._lib import BF16, F32, U8, SumDesc
from tests.gpu_util import TD
from tests.test_gpu_graph_ops import _builder_net, _frames, excess, op_class, record, sum_bound, verify_graph

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not torch.cuda.is_available(), reason="needs a CUDA device")]

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CHILD = os.environ.get("B200ROMP_SWITCH_CHILD")
LIB_SWITCHES = ("B200ROMP_SUM_RING", "B200ROMP_SUM_SIMPLE", "B200ROMP_TC_NO_FOLD", "B200ROMP_NO_PDL",
                "B200ROMP_BEV_CENTER3D_2PASS", "B200ROMP_NO_GRAPH", "B200ROMP_LANES")
BUILD_SWITCHES = ("B200ROMP_NO_SKIP_CONCAT", "B200ROMP_NO_FUSE1X1_MERGE", "B200ROMP_NO_S2_KSPLIT", "B200ROMP_S2_KSPLIT_C")
SUM_RE = re.compile(r"\[fuse-sum (\w+)\]")
CONV_RE = re.compile(r" k(\d+) s(\d) +(\d+)->(\d+) +in t\d+\[(\d+)x(\d+)x(\d+)\]\+(\d+) out t\d+\[\S+\]\+\d+ res t(-?\d+) up\d relu(\d)")


def _say(s):
    print(s, flush=True)


@pytest.fixture(scope="module")
def romp_sd():
    return synth.romp_state_dict(0)


@pytest.fixture(scope="module")
def bev_sd():
    return synth.bev_state_dict(0)


@pytest.fixture(scope="module")
def resnet50_sd():
    return synth.resnet50_state_dict(0)


def _clean_switches(monkeypatch):
    """this process must run the default library path: a switch in its own environment would have latched already"""
    for v in LIB_SWITCHES:
        if os.environ.get(v) == "1" and not CHILD:
            pytest.skip(f"{v}=1 is set for the whole run: the default path cannot be compared with its switch")
    for v in BUILD_SWITCHES:
        monkeypatch.delenv(v, raising=False)


def _plan(lines):
    """describe() op lines without op numbers and tensor ids (a switch renumbers both): a multiset of op plans"""
    return Counter(re.sub(r"t-?\d+", "t", l.split(" ", 1)[1]) for l in lines)


def _report_diff(name, default, switched):
    a, b = _plan(default), _plan(switched)
    gone, new = a - b, b - a
    _say(f"== {name}: {sum(gone.values())} op plans of the default build gone, {sum(new.values())} new")
    for l, n in sorted(gone.items()):
        _say(f"   - {n} x {l.strip()}")
    for l, n in sorted(new.items()):
        _say(f"   + {n} x {l.strip()}")
    assert gone or new, f"{name}: the switch left the plan unchanged"


def _convs(lines):
    """(ksize, stride, cin, cout, in C, in_c_off, res, relu) of every plain conv line"""
    out = []
    for l in lines:
        m = CONV_RE.search(l)
        if m and " block " not in l:
            k, s, ci, co, _, _, C_in, off, res, relu = (int(x) for x in m.groups())
            out.append(dict(k=k, s=s, cin=ci, cout=co, in_C=C_in, in_off=off, res=res, relu=relu, line=l))
    return out


def _sums(r):
    return [c[2][0] for c in r["calls"] if c[0] == "sum"]


def _producers(r):
    """tensor -> descriptor of the conv that writes it"""
    return {c[2][0].out: c[2][0] for c in r["calls"] if c[0] == "conv"}


def _sliced(r, s):
    """does sum descriptor s read a channel slice of a wider tensor?"""
    Cc = r["tensors"][s.out]["C"]
    return any(s.term_c_off[k] or r["tensors"][s.term[k]]["C"] != Cc for k in range(s.n_terms))


def _ring_takes(r, s):
    """the ring kernel's conditions (conv_simt.cu, choose_fuse_sum): every term a whole tensor, and room in shared memory
    for at least two stages of one base row plus one row of every term"""
    if _sliced(r, s):
        return False
    t = r["tensors"][s.out]
    es = 4 if t["dt"] == F32 else 2
    stage = t["W"] * t["C"] * es + sum(t["W"] // s.up[k] * t["C"] * es for k in range(s.n_terms))
    stage = -(-stage // 128) * 128
    blocks_per_sm = 3 if stage <= 21 * 1024 else 2
    return min(4, (200 * 1024 // blocks_per_sm - 256) // stage) >= 2


# ---------------------------------------------------------------------------------------------------------------------
# graph-builder switches, in this process
# ---------------------------------------------------------------------------------------------------------------------
def _build(monkeypatch, kind, sd, env):
    """-> (production net, record, its op lines, graph io) of one bf16 graph built with the variables `env` set"""
    with monkeypatch.context() as m:
        for k, v in env.items():
            m.setenv(k, v)
        if kind == "hrnet":
            (nb, io), (r,) = record(monkeypatch, lambda: graph.build_romp(sd, 0, "bf16", U8, 64))
        elif kind == "resnet50":
            (nb, io), (r,) = record(monkeypatch, lambda: graph.build_romp_resnet50(sd, 0, "bf16", U8, 64))
        else:
            (nb, io, g2, _), (r, _) = record(monkeypatch, lambda: graph.build_bev(sd, 0, "bf16", U8, 34))
            g2.lib.b200romp_net_destroy(g2.net)
    prod = _builder_net(nb, r)
    return prod, r, prod.op_lines(), io


GRAPH_BATCH = {"hrnet": 64, "resnet50": 64, "bev": 34}


def _verify_switched(name, kind, prod, r, lines, io):
    batch = GRAPH_BATCH[kind]
    frames = _frames(batch, seed=61)
    net, _, ops, _, read = verify_graph(name, r, lines, batch, {io["frames"]: frames}, _say)
    net.destroy()
    read.cache.clear()
    prod.destroy()
    return ops


SD_FIXTURE = {"hrnet": "romp_sd", "bev": "bev_sd"}


@pytest.mark.parametrize("kind", ["hrnet", "bev"])
def test_no_skip_concat(monkeypatch, request, kind):
    """layer1.0's downsample is its own 1x1 64->256 conv (no ReLU, no residual) added to conv3 as a residual, and no conv
    reads the 128-channel [conv2 | stem] concatenation"""
    _clean_switches(monkeypatch)
    sd = request.getfixturevalue(SD_FIXTURE[kind])
    p0, _, default, _ = _build(monkeypatch, kind, sd, {})
    p0.destroy()
    prod, r, lines, io = _build(monkeypatch, kind, sd, {"B200ROMP_NO_SKIP_CONCAT": "1"})
    name = f"NO_SKIP_CONCAT {kind} bf16"
    _report_diff(name, default, lines)
    cat = lambda c: c["k"] == 1 and c["cin"] == 128 and c["cout"] == 256 and c["in_C"] == 128
    down = lambda c: c["k"] == 1 and c["cin"] == 64 and c["cout"] == 256 and c["res"] < 0 and not c["relu"]
    assert any(cat(c) for c in _convs(default)) and not any(down(c) for c in _convs(default))
    assert not any(cat(c) for c in _convs(lines)), "the 128-channel concat conv is still there"
    assert sum(down(c) for c in _convs(lines)) == 1, "no separate downsample conv"
    _verify_switched(name, kind, prod, r, lines, io)


@pytest.mark.parametrize("kind", ["hrnet", "bev"])
def test_no_fuse1x1_merge(monkeypatch, request, kind):
    """one 1x1 conv per fuse term (each upsampled term of a sum is the whole output of its own 1x1 conv) and no sum reads
    a channel slice"""
    _clean_switches(monkeypatch)
    sd = request.getfixturevalue(SD_FIXTURE[kind])
    p0, r0, default, _ = _build(monkeypatch, kind, sd, {})
    p0.destroy()
    assert any(_sliced(r0, s) for s in _sums(r0)), "the default build has no merged 1x1 fuse conv"
    assert all(SUM_RE.search(l).group(1) == "pipe" for l in default if " sum " in l), "production sums left the pipe kernel"
    prod, r, lines, io = _build(monkeypatch, kind, sd, {"B200ROMP_NO_FUSE1X1_MERGE": "1"})
    name = f"NO_FUSE1X1_MERGE {kind} bf16"
    _report_diff(name, default, lines)
    assert not any(_sliced(r, s) for s in _sums(r)), "a sum still reads a channel slice"
    made_by = _producers(r)
    up_terms = [s.term[k] for s in _sums(r) for k in range(s.n_terms) if s.up[k] > 1]
    assert len(set(up_terms)) == len(up_terms), "two fuse terms share one 1x1 conv"
    for t in up_terms:
        d = made_by[t]
        assert d.ksize == 1 and d.stride == 1 and d.cout == r["tensors"][t]["C"], f"term t{t} is not a 1x1 conv of its own"
    _say(f"   {len(up_terms)} upsampled fuse terms, each from its own 1x1 conv")
    _verify_switched(name, kind, prod, r, lines, io)


def _ksplit_parts(lines):
    """the parts of the 256-channel 3x3 stride-2 conv: (cin, in_c_off) of every k3 s2 conv reading a 256-channel tensor"""
    return sorted((c["cin"], c["in_off"]) for c in _convs(lines) if c["k"] == 3 and c["s"] == 2 and c["in_C"] == 256)


@pytest.mark.parametrize("env,parts", [({"B200ROMP_NO_S2_KSPLIT": "1"}, [(256, 0)]),
                                       ({"B200ROMP_S2_KSPLIT_C": "64"}, [(64, 0), (64, 64), (64, 128), (64, 192)])],
                         ids=["NO_S2_KSPLIT", "S2_KSPLIT_C=64"])
def test_s2_ksplit(monkeypatch, resnet50_sd, env, parts):
    """ResNet-50's layer3.0 conv2 (3x3 stride 2, 256 -> 256): unsplit, on whichever engine takes it, or four 64-channel
    parts accumulating onto each other in fp32"""
    _clean_switches(monkeypatch)
    p0, _, default, _ = _build(monkeypatch, "resnet50", resnet50_sd, {})
    p0.destroy()
    assert _ksplit_parts(default) == [(128, 0), (128, 128)]
    prod, r, lines, io = _build(monkeypatch, "resnet50", resnet50_sd, env)
    name = f"{','.join(f'{k[9:]}={v}' for k, v in env.items())} ResNet-50 bf16"
    _report_diff(name, default, lines)
    assert _ksplit_parts(lines) == parts
    for c in _convs(lines):
        if c["k"] == 3 and c["s"] == 2 and c["in_C"] == 256:
            _say(f"   part: {c['line'].strip()}")
    ops = _verify_switched(name, "resnet50", prod, r, lines, io)
    assert sum(1 for op in ops if op["kind"] == "conv" and op["conv"][0].stride == 2 and op["conv"][0].ksize == 3
               and r["tensors"][op["conv"][0].in_]["C"] == 256) == len(parts)


# ---------------------------------------------------------------------------------------------------------------------
# library switches: one child process each
# ---------------------------------------------------------------------------------------------------------------------
def _pdl_outputs(romp_sd, bev_sd):
    """the outputs of the ROMP bf16 and TF32 graphs and of BEV's G1 and G2 in bf16 on seeded inputs, on the host"""
    out = {}
    stream = torch.cuda.Stream()

    def run(nb, io, batch, inputs, keys):
        binds = dict(inputs)
        for k in keys:
            s = nb.shape[io[k]]
            shape = (batch, s[2], s[0], s[1]) if k in ("center_maps", "params_maps", "maps_fv") else (batch,) + s[:3]
            binds[io[k]] = torch.zeros(shape, dtype=TD[s[3]], device="cuda")
        for t, x in binds.items():
            _lib.check(nb.lib.b200romp_net_bind(nb.net, t, x.data_ptr()), "bind")
        _lib.check(nb.lib.b200romp_net_run(nb.net, batch, stream.cuda_stream), "run")
        stream.synchronize()
        res = {k: binds[io[k]].cpu() for k in keys}
        nb.lib.b200romp_net_destroy(nb.net)
        return res

    for precision, batch in (("bf16", 64), ("tf32", 16)):
        nb, io = graph.build_romp(romp_sd, 0, precision, U8, batch)
        for k, v in run(nb, io, batch, {io["frames"]: _frames(batch, seed=71)}, ("center_maps", "params_maps")).items():
            out[f"romp_{precision}_{k}"] = v
    g1, io1, g2, io2 = graph.build_bev(bev_sd, 0, "bf16", U8, 34)
    for k, v in run(g1, io1, 34, {io1["frames"]: _frames(34, seed=72)}, ("maps_fv", "fv_feats", "img_feats")).items():
        out[f"bev_g1_{k}"] = v
    g = torch.Generator(device="cuda").manual_seed(73)
    bv = torch.randn(34, 1, 128, 2560, generator=g, device="cuda").abs().bfloat16()
    out["bev_g2_bv_out"] = run(g2, io2, 34, {io2["bv_in"]: bv}, ("bv_out",))["bv_out"]
    return out


CHILDREN = {
    "SUM_SIMPLE": {"B200ROMP_SUM_SIMPLE": "1"},
    "SUM_RING": {"B200ROMP_SUM_RING": "1"},
    "SUM_RING_NO_FUSE1X1_MERGE": {"B200ROMP_SUM_RING": "1", "B200ROMP_NO_FUSE1X1_MERGE": "1"},
    "TC_NO_FOLD": {"B200ROMP_TC_NO_FOLD": "1"},
    "NO_PDL": {"B200ROMP_NO_PDL": "1"},
    "BEV_CENTER3D_2PASS": {"B200ROMP_BEV_CENTER3D_2PASS": "1"},
}
CHILD_TEST = {"SUM_SIMPLE": "test_child_sum", "SUM_RING": "test_child_sum", "SUM_RING_NO_FUSE1X1_MERGE": "test_child_sum",
              "TC_NO_FOLD": "test_child_tc_no_fold", "NO_PDL": "test_child_no_pdl",
              "BEV_CENTER3D_2PASS": "test_child_center3d_2pass"}


@pytest.mark.parametrize("name", list(CHILDREN))
def test_library_switch(monkeypatch, tmp_path, romp_sd, bev_sd, name):
    """runs the child test of one library switch in a fresh process with the switch in its environment"""
    if CHILD:
        pytest.skip("inside a child")
    _clean_switches(monkeypatch)
    if name == "NO_PDL":
        torch.save(_pdl_outputs(romp_sd, bev_sd), tmp_path / "default_outputs.pt")
        torch.cuda.empty_cache()
    env = {k: v for k, v in os.environ.items() if k not in LIB_SWITCHES + BUILD_SWITCHES}
    env.update(CHILDREN[name])
    env["B200ROMP_SWITCH_CHILD"] = name
    env["B200ROMP_SWITCH_REF"] = str(tmp_path / "default_outputs.pt")
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [
        "-m", "pytest", f"{os.path.abspath(__file__)}::{CHILD_TEST[name]}", "-s", "-q", "-p", "no:cacheprovider"]
    t0 = time.time()
    p = subprocess.run(cmd, env=env, cwd=ROOT, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=1200)
    dt = time.time() - t0
    _say(f"######## child {name} ({' '.join(f'{k}={v}' for k, v in CHILDREN[name].items())}): exit {p.returncode}, "
         f"{dt:.1f} s\n{p.stdout}")
    assert p.returncode == 0, f"child {name} failed (exit {p.returncode}):\n{p.stdout[-6000:]}"
    assert re.search(r"\b1 passed\b", p.stdout) and "skipped" not in p.stdout, f"child {name} did not run its test"


def _child(name_prefix):
    if not CHILD or not CHILD.startswith(name_prefix):
        pytest.skip("runs only in the child process of test_library_switch")


# ---- fuse-sum kernels ------------------------------------------------------------------------------------------------
SUM_SHAPES = [(32, 32, 32, [2, 4, 8]), (16, 16, 64, [1, 2]), (8, 8, 256, [1]), (128, 128, 32, [2, 4, 8]), (32, 96, 32, [2])]


def _standalone_sum(dtype, H, W, Cc, ups):
    """one sum op of external tensors -> (worst |err|/bound vs float64, bit-equal to the fp32 sum in kernel order,
    the kernel describe() names once bound)"""
    lib = _lib.load()
    dev = torch.device("cuda", 0)
    B = 3
    g = torch.Generator().manual_seed(H * 7 + W + Cc)
    base = torch.randn(B, H, W, Cc, generator=g).to(dev, TD[dtype])
    terms = [torch.randn(B, H // u, W // u, Cc, generator=g).to(dev, TD[dtype]) for u in ups]
    out = torch.full((B, H, W, Cc), float("nan"), dtype=TD[dtype], device=dev)
    net = lib.b200romp_net_create(0)
    try:
        tb = lib.b200romp_net_add_tensor(net, H, W, Cc, dtype, 0, 1)
        tt = [lib.b200romp_net_add_tensor(net, H // u, W // u, Cc, dtype, 0, 1) for u in ups]
        to = lib.b200romp_net_add_tensor(net, H, W, Cc, dtype, 0, 1)
        d = SumDesc(to, tb, len(ups), (C.c_int * 4)(*(tt + [0] * (4 - len(tt)))), (C.c_int * 4)(*(ups + [1] * (4 - len(ups)))), 1)
        _lib.check(lib.b200romp_net_add_sum(net, C.byref(d)), "add_sum")
        _lib.check(lib.b200romp_net_finalize(net, B), "finalize")
        for t, x in zip([tb] + tt + [to], [base] + terms + [out]):
            _lib.check(lib.b200romp_net_bind(net, t, x.data_ptr()), "bind")
        buf = C.create_string_buffer(1 << 12)
        lib.b200romp_net_describe(net, buf, len(buf))
        kernel = SUM_RE.search(buf.value.decode()).group(1)
        _lib.check(lib.b200romp_net_run(net, B, torch.cuda.current_stream().cuda_stream), "run")
        torch.cuda.synchronize()
    finally:
        lib.b200romp_net_destroy(net)
    v, bnd = sum_bound(base.double(), [t.double() for t in terms], ups, True, dtype)
    worst, over = excess(out, v, bnd)
    ref = base.float()
    for t, u in zip(terms, ups):
        ref = ref + t.float().repeat_interleave(u, 1).repeat_interleave(u, 2)
    exact = torch.equal(out, ref.clamp_min(0).to(TD[dtype]))
    return worst, over, exact, kernel


def test_child_sum(monkeypatch, romp_sd):
    _child("SUM_")
    want = "simple" if CHILD == "SUM_SIMPLE" else "ring"
    bad = []
    for dtype in (F32, BF16):
        for H, W, Cc, ups in SUM_SHAPES:
            worst, over, exact, kernel = _standalone_sum(dtype, H, W, Cc, ups)
            what = f"sum {'fp32' if dtype == F32 else 'bf16'} {H}x{W}x{Cc} ups {ups}"
            _say(f"   {what}: [fuse-sum {kernel}], worst |err|/bound {worst:.3f}, bit-equal to the fp32 sum {exact}")
            if kernel != want or over or not exact:
                bad.append(f"{what}: kernel {kernel} (want {want}), {over} elements over the bound, bit-equal {exact}")
    assert not bad, "\n".join(bad)
    # every sum op of the ROMP graphs, in place
    merged = os.environ.get("B200ROMP_NO_FUSE1X1_MERGE") != "1"
    for precision, batch in (("bf16", 64), ("tf32", 34)):
        (nb, io), (r,) = record(monkeypatch, lambda: graph.build_romp(romp_sd, 0, precision, U8, batch))
        prod = _builder_net(nb, r)
        lines = prod.op_lines()
        name = f"{CHILD} ROMP {precision}"
        net, _, ops, _, read = verify_graph(name, r, lines, batch, {io["frames"]: _frames(batch, seed=62)}, _say)
        net.destroy()
        read.cache.clear()
        prod.destroy()
        took, wrong = Counter(), []
        for op in ops:
            if op["kind"] != "sum":
                continue
            kernel = SUM_RE.search(op["line"]).group(1)
            took[kernel] += 1
            # the ring kernel takes a sum of whole tensors whose rows fit its stages; with the merged 1x1 convs a sum may
            # read channel slices, and fp32 rows of 256 channels or of 128 channels and three terms leave room for one stage
            expect = want if (want == "simple" or _ring_takes(r, op["sum"])) else "pipe"
            if kernel != expect:
                wrong.append(f"{op['line'].strip()}: want {expect}")
        _say(f"   {name}: sum ops by kernel {dict(took)}" + ("" if merged else " (unmerged 1x1 fuse convs)"))
        assert not wrong, "sum ops on the wrong kernel:\n" + "\n".join(wrong)
        assert took[want] > 0


# ---- unfolded 32-channel convs ---------------------------------------------------------------------------------------
def test_child_tc_no_fold(monkeypatch, romp_sd):
    _child("TC_NO_FOLD")
    from tests import test_gpu_conv_tc as tc
    cases = [c for c in tc.CASES if c[2] == 32 and c[3] == 32]
    for case in cases:
        tc.test_tcgen05_conv_matches_torch(case)
        _say(f"   test_gpu_conv_tc {case[0]}: within tolerance")
    (nb, io), (r,) = record(monkeypatch, lambda: graph.build_romp(romp_sd, 0, "bf16", U8, 64))
    prod = _builder_net(nb, r)
    lines = prod.op_lines()
    text = "\n".join(lines)
    assert "pixel-pairs" not in text, "a conv still runs pixel-pair folded"
    assert not re.search(r"block k3 s1 32->32->32", text), "a 32-channel BasicBlock still runs fused"
    n32 = sum(1 for c in _convs(lines) if c["k"] == 3 and c["s"] == 1 and c["cin"] == 32 and c["cout"] == 32 and "[tc" in c["line"])
    _say(f"   TC_NO_FOLD: {n32} unfolded 32->32 3x3 convs on the tensor-core engine, no pixel-pair fold, no fused 32-channel block")
    assert n32 >= 64
    net, _, ops, _, read = verify_graph("TC_NO_FOLD ROMP bf16", r, lines, 64, {io["frames"]: _frames(64, seed=63)}, _say)
    assert {"block", "folded block"} & {op_class(op) for op in ops} == {"block"}
    net.destroy()
    read.cache.clear()
    prod.destroy()


# ---- programmatic dependent launch off ----------------------------------------------------------------------------
def test_child_no_pdl(romp_sd, bev_sd):
    _child("NO_PDL")
    # tc_launch latches the variable at its first launch: it must have come with the process, before the library loaded
    assert os.environ.get("B200ROMP_NO_PDL") == "1" and _lib._lib is None
    ref = torch.load(os.environ["B200ROMP_SWITCH_REF"])
    got = _pdl_outputs(romp_sd, bev_sd)
    assert sorted(got) == sorted(ref)
    diff = [k for k in ref if not torch.equal(got[k], ref[k])]
    for k in sorted(ref):
        _say(f"   NO_PDL {k} {tuple(ref[k].shape)}: {'DIFFERS' if k in diff else 'bit-identical'} to the default (PDL) run")
    assert not diff, f"outputs differ without programmatic dependent launch: {diff}"


# ---- two-pass 3-D centre map ---------------------------------------------------------------------------------------
def test_child_center3d_2pass(bev_sd):
    _child("BEV_CENTER3D_2PASS")
    from tests import test_gpu_bev_detect_fp64 as D
    sd64 = {k: torch.from_numpy(np.asarray(v)).to("cuda", torch.float64) for k, v in bev_sd.items()
            if k.startswith(("center_map_refiner.", "cam_map_refiner.", "transformer.", "position_embeddings.", "coordmap_3d"))}

    def check(m, maps_fv, bv, code, name):
        tmp = m.buf["c3d_tmp"]
        tmp.fill_(float("nan"))
        D.check_center3d(m, sd64, maps_fv, bv, code, name)
        n = maps_fv.shape[0]
        assert torch.isfinite(tmp[:n]).all(), f"{name}: the two-pass kernel did not write its intermediate"
        assert torch.isnan(tmp[n:]).all(), f"{name}: the intermediate spills past frame {n}"

    for precision in ("fp32", "bf16"):
        m = D.model(bev_sd, precision)
        frames = torch.from_numpy(synth.synthetic_frames(3, seed=11)).to("cuda")
        with torch.cuda.stream(m.stream):
            m.run_model(frames)
        m.stream.synchronize()
        b = m.buf
        check(m, b["maps_fv"][:3], b["bv_out"][:3], D.ACT[precision][1], f"2-pass model {precision}")
        for batch in (1, 3, 32):
            maps_fv, bv, _ = D.crafted_maps(batch, 100 + batch, D.ACT[precision][0])
            check(m, maps_fv, bv, D.ACT[precision][1], f"2-pass crafted {precision} B={batch}")
