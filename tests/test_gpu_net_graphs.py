"""Seeded random conv graphs (tests/net_graphs.py) checked op by op against float64, and the aliasing rule of the graph
calls.

test_generated_graphs takes every seed of net_graphs.SEEDS through test_gpu_graph_ops.verify_graph at net_graphs.BATCH:
the keeper net, every op within the float64 bound of that file, and ops whose tiles cannot give some CTA a third tile
rerun alone at a batch that does.  Then, per seed, bits are compared:
  - the production net (buffer reuse) against the keeper net, on every external output;
  - the keeper net at batch 1 (fewer tiles than CTAs for every persistent op) and inside a batch of 7, on every tensor
    it keeps and every external output, against the same frames of the graph batch;
  - B200ROMP_NO_GRAPH=1 (eager launches) and B200ROMP_LANES=1 (ops on their lanes' streams) against the default net;
  - on seed 0, 18 distinct bindings of every external tensor, which makes the 16-entry CUDA-graph cache clear itself.
The plan of every op is read from describe(): each planted op must get the plan it was planted for, and across the
seeds every item of the coverage table must be reached (a missing item fails the test; the remedy is a planted case).
The workspace size must equal net_graphs.plan_workspace, the buffer planner restated on describe()'s op list, and some
buffer must be recycled between ops of different lanes.  negative_controls of test_gpu_graph_ops run on the first seed
that has the ops they mutate.

The aliasing tests: every rejected form returns B200ROMP_EINVAL with its message; the identical-slice forms (a residual
that is the output slice, a disjoint output slice of the input tensor) compute the float64 result; an in-place
BasicBlock and an in-place Bottleneck are not fused (describe()) and are correct.

Measured on one H100 80GB HBM3 at a 700 W power limit: 160 seeds, 1770 ops in 29 s (test_generated_graphs), the whole
file 40 s; peak torch allocation of any seed 3.6 GiB (keeper-net workspaces, at most 0.1 GiB, not counted).
"""
import ctypes as C
import math
import re
import time

import numpy as np
import pytest
import torch

from romp_b200 import _lib
from romp_b200._lib import BF16, ENGINE_AUTO, F32, U8, ConvDesc
from tests import net_graphs as NG
from tests.gpu_util import TD
from tests.test_gpu_graph_ops import (TC_RE, Net, block_bound, conv_bound, excess, internal_tensors, negative_controls, ops_of,
                                      tiles_per_cta, verify_graph)


def _say(s):
    print(s, flush=True)


# ---------------------------------------------------------------------------------------------------------------------
# what describe() says each op runs
# ---------------------------------------------------------------------------------------------------------------------
def _simt_inst(d, T):
    """the CUDA-core kernel launch_conv_simt / choose_kernel run for a conv descriptor"""
    if d.ksize == 7:
        return "k7"
    if d.ksize == 42:
        return "deconv"
    to = T[d.out]
    if (d.ksize == 3 and d.stride == 2 and d.cin == 3 and d.cout <= 64 and d.cout % 16 == 0 and not to["nchw"] and d.res < 0
            and d.upsample == 1 and d.pow_channel < 0 and to["C"] % 8 == 0 and d.out_c_off % 8 == 0):
        return "stem"
    if d.ksize == 13:
        return "131"
    return f"{d.ksize}{d.ksize}{d.stride}"


def plans(r, lines):
    """-> per describe() op line: dict(ids = recorded op ids, plan = the plan tuple, op = ops_of entry)"""
    T = r["tensors"]
    calls = [c for c in r["calls"] if c[0] in ("conv", "sum", "maxpool")]
    out, i = [], 0
    for op in ops_of(r, lines):
        n = 2 if op["kind"] == "block" else 1
        ids = tuple(c[1] for c in calls[i:i + n])
        i += n
        if op["kind"] == "block":
            plan = ("block", op["fold"])
        elif op["kind"] == "sum":
            m = re.search(r"\[fuse-sum (\w+)\]", op["line"])
            plan = ("sum", m.group(1), T[op["sum"].base]["dt"])
        elif op["kind"] == "maxpool":
            plan = ("maxpool", T[op["io"][0]]["dt"])
        else:
            d, tc = op["conv"][0], op["tc"]
            if tc is None:
                plan = ("simt", _simt_inst(d, T))
            elif "bottleneck" in tc:
                plan = ("bottleneck", tc["bottleneck"])
            else:
                m = TC_RE.search(op["line"])
                kind, nt, eb = int(m.group(2)) * 10 + int(m.group(3)), int(m.group(4)), 4 if m.group(1) else 2
                f = 2 if tc["fold"] else 1
                generic = not ((d.cout * f) % nt == 0 and d.upsample == 1 and not T[d.out]["nchw"] and d.pow_channel < 0)
                mode = 2 if kind == 32 else kind // 10
                plan = ("tc", kind, mode, d.cin * f, nt, eb, generic)
        out.append(dict(ids=ids, plan=plan, op=op, num=int(op["line"][2:5])))
    return out


def stored_mids(r, p):
    """the Bottleneck intermediates that ops outside the chain read"""
    groups = {}
    for e in p:
        if e["plan"][0] == "bottleneck":
            groups.setdefault(e["num"], []).append(e)
    stored = {}
    for num, es in groups.items():
        ids = {e["ids"][0] for e in es}
        mids = [e["op"]["conv"][0].out for e in es[:-1]]
        readers = set()
        for kind, op, args in r["calls"]:
            if op in ids:
                continue
            if kind == "conv":
                readers |= {args[0].in_, args[0].res}
            elif kind == "sum":
                readers |= {args[0].base} | {args[0].term[k] for k in range(args[0].n_terms)}
            elif kind == "maxpool":
                readers.add(args[0])
        stored[num] = [m for m in mids if m in readers]
    return stored


def planner_ops(r, p, lanes):
    """describe()'s ops as net_graphs.plan_workspace takes them: a fused op reads its first conv's input and writes its
    output and the intermediates other ops read"""
    T = r["tensors"]
    stored = stored_mids(r, p)
    ops, seen = [], {}
    for e in p:
        op = e["op"]
        if e["num"] in seen:
            continue
        seen[e["num"]] = True
        if op["kind"] == "sum":
            s = op["sum"]
            ops.append(dict(reads=[s.base] + [s.term[k] for k in range(s.n_terms)], writes=[s.out], lane=lanes.get(e["ids"][0], 0)))
        elif op["kind"] == "maxpool":
            ops.append(dict(reads=[op["io"][0]], writes=[op["io"][1]], lane=lanes.get(e["ids"][0], 0)))
        elif op["kind"] == "block":
            d1, d2 = op["convs"][0][0], op["convs"][1][0]
            ops.append(dict(reads=[d1.in_], writes=[d2.out], lane=lanes.get(e["ids"][0], 0)))
        elif e["plan"][0] == "bottleneck":
            parts = [x for x in p if x["num"] == e["num"]]
            d1, d3 = parts[0]["op"]["conv"][0], parts[-1]["op"]["conv"][0]
            ops.append(dict(reads=[d1.in_], writes=[d3.out] + stored[e["num"]], lane=lanes.get(e["ids"][0], 0)))
        else:
            d = op["conv"][0]
            ops.append(dict(reads=[d.in_] + ([d.res] if d.res >= 0 else []), writes=[d.out], lane=lanes.get(e["ids"][0], 0)))
    return [o for o in ops], {k: v for k, v in T.items()}


def expected_ok(plan, expect, stored):
    kind = expect[0]
    if kind == "tc":
        return plan[0] == "tc" and plan[1] in (10, 30, 32) and plan[2:] == expect[1]
    if kind == "kind":
        return plan[0] == "tc" and plan[1] == expect[1]
    if kind == "simt":
        return plan == ("simt", expect[1])
    if kind == "maxpool":
        return plan == ("maxpool", expect[1])
    if kind == "sum":
        return plan[:2] == ("sum", expect[1])
    if kind == "block":
        return plan == ("block", expect[1])
    if kind == "bottleneck":
        return plan[0] == "bottleneck" and bool(stored) == expect[1]
    raise AssertionError(expect)


# ---------------------------------------------------------------------------------------------------------------------
# the coverage table
# ---------------------------------------------------------------------------------------------------------------------
def coverage_items():
    src = open(NG.__file__.replace("tests/net_graphs.py", "romp_b200/csrc/conv_tc.cu")).read()
    rows = NG.b2r_rows(src)
    dead = set(NG.unreachable_rows(rows))
    items = []
    for (mode, cin, nt, eb) in rows:
        if (mode, cin, nt, eb) in dead:
            continue
        for generic in (False, True):
            items.append(("tc row", (mode, cin, nt, eb, generic)))
    items += [("kind", k) for k in (31, 34, 33, 13)]
    items += [("block", f) for f in (False, True)] + [("bottleneck", s) for s in (False, True)]
    items += [("simt", i) for i in ("stem", "131", "331", "332", "111", "112", "k7", "deconv")]
    items += [("maxpool", dt) for dt in (BF16, F32)]
    items += [("sum", k, dt) for k in ("pipe", "simple") for dt in (BF16, F32)]
    items += [("tiles >= 3", f) for f in ("conv", "swap", "stream", "stem", "conv1d", "block", "bottleneck")]
    items += [("tiles < CTAs", f) for f in ("conv", "swap", "stream", "stem", "conv1d", "block", "bottleneck")]
    items += [("SIMT fallback", w) for w in ("cin 48", "cout 48", "height 40", "width 20", "stride-2 height 24", "in_c_off 4",
                                              "tf32 with bf16 residual", "tf32 256-channel stride 2", "external input")]
    items += [("near miss", w) for w in ("block: intermediate external", "block: second reader", "block: different lanes",
                                          "block: residual from another slice", "block: no ReLU", "block: odd side",
                                          "bottleneck: intermediate external", "bottleneck: different lanes",
                                          "bottleneck: no ReLU")]
    items += [("buffer recycled across lanes", None)]
    return items, dead


def family(plan):
    if plan[0] == "tc":
        return {31: "swap", 34: "stream", 33: "stem", 13: "conv1d"}.get(plan[1], "conv")
    if plan[0] in ("block", "bottleneck"):
        return plan[0]
    return None


def covered_by(r, p, stored, batch):
    """coverage items the op lines of one graph reach (the tile items at the graph batch and at batch 1)"""
    got = set()
    for e in p:
        plan = e["plan"]
        if plan[0] == "tc":
            if plan[1] in (10, 30, 32):
                got.add(("tc row", plan[2:]))
            else:
                got.add(("kind", plan[1]))
        elif plan[0] == "bottleneck":
            got.add(("bottleneck", bool(stored.get(e["num"]))))
        elif plan[0] == "sum":
            got.add(("sum", plan[1], plan[2]))
        else:
            got.add(plan)
        fam = family(plan)
        if fam:
            op = e["op"]
            grid = op["grid"] if op["kind"] == "block" else op["tc"]["grid"]
            n_b = tiles_per_cta(op, r["tensors"], batch)[0]
            n_1 = tiles_per_cta(op, r["tensors"], 1)[1]
            if n_b is None and fam == "bottleneck":      # per conv of the chain: 16x8 tiles of the block's output
                T = r["tensors"][op["conv"][0].out]
                n_1 = (T["H"] // 16) * (T["W"] // 8)
                n_b = -(-n_1 * batch // min(grid, n_1 * batch))
            if fam == "stream":                           # 16x16 tiles, one work item per 64-channel slab
                d = op["conv"][0]
                T = r["tensors"][d.out]
                n_1 = (T["H"] // 16) * (T["W"] // 16) * (d.cout // 64)
                n_b = -(-n_1 * batch // min(grid, n_1 * batch))
            if n_b is not None and n_b >= 3:
                got.add(("tiles >= 3", fam))
            if n_1 is not None and n_1 < grid:
                got.add(("tiles < CTAs", fam))
    return got


# ---------------------------------------------------------------------------------------------------------------------
# the generated graphs
# ---------------------------------------------------------------------------------------------------------------------
def make_inputs(r, g, batch, seed):
    gen = torch.Generator(device="cuda").manual_seed(1000 + seed)
    out = {}
    for t in g.inputs:
        s = r["tensors"][t]
        shape = (batch, s["H"], s["W"], s["C"])
        if s["dt"] == U8:
            out[t] = torch.randint(0, 256, shape, generator=gen, device="cuda", dtype=torch.uint8)
        else:
            out[t] = torch.randn(shape, generator=gen, device="cuda").to(TD[s["dt"]])
    return out


def ext_outputs(r, g):
    return [t for t, s in r["tensors"].items() if s["ext"] and t not in g.inputs]


def run_net(net, r, g, batch, inputs, stream, extra=None):
    """run `net` at `batch` on the first `batch` frames of `inputs`; -> its external outputs (fresh zeroed buffers)"""
    binds = {t: inputs[t][:batch].contiguous() for t in g.inputs}
    outs = {t: net.alloc(t, batch).zero_() for t in ext_outputs(r, g)}
    with torch.cuda.stream(stream):
        net.run(batch, {**binds, **outs, **(extra or {})}, stream)
    stream.synchronize()
    return outs


def _has_control_ops(r):
    """the graph has the ops negative_controls needs: a stride-2 1x1 or 3x3 conv of activations and a conv with a
    batched residual of >= 8 channels"""
    T = r["tensors"]
    convs = [a[0] for k, _, a in r["calls"] if k == "conv"]
    return any(d.stride == 2 and d.ksize in (1, 3) and T[d.in_]["dt"] != U8 for d in convs) and any(
        d.res >= 0 and d.cout >= 8 and not d.res_broadcast for d in convs)


def _check_seed(monkeypatch, seed, cov, lane_recycle, report, controls):
    g = NG.generate(seed)
    r = g.record()
    B = r["max_batch"]
    prod = Net.replay(r)
    lines = prod.op_lines()
    p = plans(r, lines)
    stored = stored_mids(r, p)

    # planted ops got their plans
    by_id = {}
    for e in p:
        for i in e["ids"]:
            by_id.setdefault(i, []).append(e)
    for item, ids, expect in g.expect:
        es = [e for i in ids for e in by_id[i]]
        if expect[0] == "unfused":
            assert all(e["plan"][0] not in ("block", "bottleneck") for e in es) and len({e["num"] for e in es}) == len(ids), \
                f"seed {seed}: {item} was fused:\n" + "\n".join(e["op"]["line"] for e in es)
            cov.add(("near miss", item.replace(" near miss", "")))
            continue
        e = es[0]
        st = stored.get(e["num"])
        assert expected_ok(e["plan"], expect, st), f"seed {seed}: {item} got {e['plan']}:\n{e['op']['line']}"
        if item.startswith("SIMT fallback: "):
            cov.add(("SIMT fallback", item.split(": ")[1]))
    cov.update(covered_by(r, p, stored, B))

    # the buffer planner, restated
    lanes = {op: lane for kind, _, args in r["calls"] if kind == "lane" for op, lane in [args]}
    pops, T = planner_ops(r, p, lanes)
    total, bufs = NG.plan_workspace(T, pops, B)
    ws = prod.lib.b200romp_net_workspace_bytes(prod.net)
    assert total == ws, f"seed {seed}: restated planner {total} B, library {ws} B"
    for b in bufs:
        ls = [pops[i]["lane"] for _, i in b["held"]]
        if any(a != c for a, c in zip(ls, ls[1:])):
            lane_recycle.append(seed)
            cov.add(("buffer recycled across lanes", None))
            break

    inputs = make_inputs(r, g, B, seed)
    net, binds, ops, stream, read = verify_graph(f"seed {seed}", r, lines, B, inputs, report)
    if controls:
        negative_controls(ops, read, B, report)
    outs = ext_outputs(r, g)
    kept_out = {t: binds[t] for t in outs}
    kept_int = {t: read(t) for t in _kept(r, lines)}
    read.cache.clear()

    # keeper net at batch 1 and inside a batch of 7: every kept tensor, every external output
    sizes = [net.alloc(k, 1).nbytes for k in net.keepers] or [1]
    scratch = torch.empty(max(sizes) * 7, dtype=torch.uint8, device="cuda")
    kb = {k: scratch for k in net.keepers}
    for i in (0, B - 1):
        lo = min(max(i - 3, 0), B - 7)
        for n, first in ((1, i), (7, lo)):
            sub = {t: v[first:first + n] for t, v in inputs.items()}
            got = run_net(net, r, g, n, sub, stream, kb)
            for t in outs:
                assert torch.equal(got[t], kept_out[t][first:first + n]), f"seed {seed}: output t{t} at batch {n} differs"
            for t, v in kept_int.items():
                assert torch.equal(net.read(t, n, stream), v[first:first + n]), \
                    f"seed {seed}: t{t} at batch {n} differs from batch {B}"
    del scratch, kb
    net.destroy()

    # buffer reuse, eager launches, lanes
    got = run_net(prod, r, g, B, inputs, stream)
    for t in outs:
        assert torch.equal(got[t], kept_out[t]), f"seed {seed}: production net output t{t} differs from the keeper net"
    for env in ("B200ROMP_NO_GRAPH", "B200ROMP_LANES"):
        with monkeypatch.context() as m:
            m.setenv(env, "1")
            other = Net.replay(r)
        assert other.op_lines() == lines
        got = run_net(other, r, g, B, inputs, stream)
        other.destroy()
        for t in outs:
            assert torch.equal(got[t], kept_out[t]), f"seed {seed}: {env}=1 output t{t} differs"
    if seed == 0:
        alive = []
        for j in range(18):
            sub = {t: v[j:j + 2].clone() for t, v in inputs.items()}
            got = run_net(prod, r, g, 2, sub, stream)
            alive.append((sub, got))
            for t in outs:
                assert torch.equal(got[t], kept_out[t][j:j + 2]), f"seed {seed}: binding {j} after the graph cache cycled"
    prod.destroy()
    return len(lines)


def _kept(r, lines):
    mids = {int(m.group(1)) for l in lines for m in [re.search(r"mid t(\d+)", l)] if m}
    return internal_tensors(r, mids)


@pytest.mark.gpu
def test_generated_graphs(monkeypatch):
    t0 = time.time()
    cov, lane_recycle, n_ops, controls, peak = set(), [], 0, None, 0
    for seed in NG.SEEDS:
        r = NG.generate(seed).record()
        ctl = controls is None and _has_control_ops(r)
        controls = seed if ctl else controls
        n_ops += _check_seed(monkeypatch, seed, cov, lane_recycle, _say if ctl else (lambda s: None), ctl)
        peak = max(peak, torch.cuda.max_memory_allocated())       # verify_graph resets the peak per seed
    assert controls is not None, "no seed has the ops the negative controls mutate"
    items, dead = coverage_items()
    lines = [f"== {len(NG.SEEDS)} seeds, {n_ops} ops, {time.time() - t0:.1f} s, peak torch memory {peak / 2**30:.2f} GiB; "
             f"B2R_CASE rows no shape selects: {sorted(dead)}"]
    missing = []
    for it in items:
        ok = it in cov
        missing += [] if ok else [it]
        lines.append(f"   {'reached' if ok else 'MISSING':8s} {it[0]:30s} {it[1:]}")
    _say("\n".join(lines))
    assert not missing, f"coverage items no seed reaches: {missing}"


# ---------------------------------------------------------------------------------------------------------------------
# the aliasing rule
# ---------------------------------------------------------------------------------------------------------------------
def _desc(i, o, cin, cout, k=3, in_off=0, out_off=0, res=-1, res_off=0, bcast=0, relu=1):
    return ConvDesc(i, in_off, o, out_off, res, res_off, bcast, cin, cout, k, 1, relu, 1, 0, -1, ENGINE_AUTO)


def _w(rng, cout, cin, k):
    return NG.bf16_round(rng.standard_normal(cout * cin * k * k) * (1.2 / math.sqrt(cin * k * k)))


@pytest.mark.gpu
def test_aliasing_rejected():
    lib = _lib.load()
    net = lib.b200romp_net_create(0)
    try:
        x = lib.b200romp_net_add_tensor(net, 32, 32, 128, BF16, 0, 0)
        c = lib.b200romp_net_add_const_tensor(net, 32, 32, 64, F32, np.zeros(32 * 32 * 64, np.float32).ctypes.data_as(C.c_void_p))
        p1 = lib.b200romp_net_add_tensor(net, 1, 1, 16, BF16, 0, 0)
        w = np.ones(128 * 128 * 9, np.float32)
        wp = w.ctypes.data_as(C.POINTER(C.c_float))
        for what, d, msg in (
                ("3x3 input slice over the output slice", _desc(x, x, 64, 64, 3, 0, 32), "input slice [0, 64) of tensor"),
                ("1x1 in place", _desc(x, x, 64, 64, 1, 0, 0), "overlaps the output slice [0, 64)"),
                ("1x1 output inside the input slice", _desc(x, x, 128, 32, 1, 0, 64), "input slice [0, 128)"),
                ("residual shifted by 8 channels", _desc(x, x, 32, 64, 1, 0, 64, x, 56), "residual slice [56, 120)"),
                ("residual partly over the output", _desc(x, x, 32, 32, 1, 32, 64, x, 80), "residual slice [80, 112)"),
                ("broadcast residual that is the output slice", _desc(x, x, 32, 32, 1, 0, 64, x, 64, 1), "without being it")):
            rc = lib.b200romp_net_add_conv(net, C.byref(d), wp, None)
            err = lib.b200romp_last_error().decode()
            assert rc == -1 and msg in err, (what, rc, err)
        rc = lib.b200romp_net_add_maxpool(net, p1, p1)
        assert rc == -1 and "is the output tensor" in lib.b200romp_last_error().decode()
        # the allowed forms: a disjoint output slice of the input tensor, a residual that is the output slice
        ok = [_desc(x, x, 64, 64, 1, 0, 64), _desc(x, x, 32, 32, 3, 0, 96, x, 96), _desc(x, x, 64, 32, 1, 64, 0, c, 0, 1)]
        for d in ok:
            assert lib.b200romp_net_add_conv(net, C.byref(d), wp, None) >= 0, lib.b200romp_last_error().decode()
    finally:
        lib.b200romp_net_destroy(net)


def _identity(lib, net, src, dst, Cc):
    eye = np.eye(Cc, dtype=np.float32).reshape(-1)
    d = _desc(src, dst, Cc, Cc, 1, relu=0)
    d.engine = _lib.ENGINE_SIMT
    _lib.check(lib.b200romp_net_add_conv(net, C.byref(d), eye.ctypes.data_as(C.POINTER(C.c_float)), None), "copy")


def _inplace_graph(kind, seed=0):
    """x (internal, written by a 1x1 conv of an external input), a copy of x, then the in-place chain: a BasicBlock
    relu(conv2(relu(conv1(x))) + x) with 64 channels (or 32 pixel-pair foldable ones), a Bottleneck of 256 -> 64 -> 64 ->
    256, or a single 3x3 conv whose residual is its output slice, written back into x.  -> (net, tensors, convs, io)"""
    rng = np.random.default_rng(seed)
    lib = _lib.load()
    net = lib.b200romp_net_create(0)
    T = {}

    def tensor(H, W, Cc, ext=0):
        t = _lib.check(lib.b200romp_net_add_tensor(net, H, W, Cc, BF16, 0, ext))
        T[t] = dict(H=H, W=W, C=Cc, dt=BF16, nchw=0, ext=ext, const=False)
        return t

    Cx = {"block": 64, "block32": 32, "bottleneck": 256, "conv": 64}[kind]
    src = tensor(64, 64, 16, ext=1)
    x = tensor(64, 64, Cx)
    keep = []
    convs = []

    def conv(d, k, b=True):
        w = _w(rng, d.cout, d.cin, k)
        bias = (0.1 * rng.standard_normal(d.cout)).astype(np.float32) if b else None
        _lib.check(lib.b200romp_net_add_conv(net, C.byref(d), w.ctypes.data_as(C.POINTER(C.c_float)),
                                             None if bias is None else bias.ctypes.data_as(C.POINTER(C.c_float))), "conv")
        convs.append((d, w, bias))

    conv(_desc(src, x, 16, Cx, 1), 1)
    convs.clear()
    x0 = tensor(64, 64, Cx)
    _identity(lib, net, x, x0, Cx)
    if kind in ("block", "block32"):
        t = tensor(64, 64, Cx)
        conv(_desc(x, t, Cx, Cx, 3), 3)
        conv(_desc(t, x, Cx, Cx, 3, res=x), 3)
        mids = [t]
    elif kind == "bottleneck":
        t1, t2 = tensor(64, 64, 64), tensor(64, 64, 64)
        conv(_desc(x, t1, 256, 64, 1), 1)
        conv(_desc(t1, t2, 64, 64, 3), 3)
        conv(_desc(t2, x, 64, 256, 1, res=x), 1)
        mids = [t1, t2]
    else:
        t = tensor(64, 64, 64)
        conv(_desc(x0, t, 64, 64, 1), 1)
        conv(_desc(t, x, 64, 64, 3, res=x), 3)
        mids = [t]
    # copies that keep x and the Bottleneck's intermediates readable after the run (a block's intermediate gets none: a
    # second reader would keep the block from fusing)
    if kind != "bottleneck":
        mids = [m for m in mids if kind == "conv"]
    outs = []
    for m in mids + [x, x0]:
        k = tensor(64, 64, T[m]["C"], ext=1)
        _identity(lib, net, m, k, T[m]["C"])
        outs.append(k)
    _lib.check(lib.b200romp_net_finalize(net, 20), "finalize")
    return Net(lib, net, T, 20), convs, dict(src=src, x=x, x0=x0, mids=mids, outs=outs)


def run_inplace(kind):
    """build and run the in-place graph of `kind`; -> (describe() op lines, worst |err|/bound, [failures])"""
    net, convs, io = _inplace_graph(kind)
    lines = net.op_lines()
    B = net.max_batch
    gen = torch.Generator(device="cuda").manual_seed(3)
    frames = torch.randn(B, 64, 64, 16, generator=gen, device="cuda").bfloat16()
    vals = {io["src"]: frames}
    for k in io["outs"]:
        vals[k] = net.alloc(k, B).zero_()
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        net.run(B, vals, stream)
    stream.synchronize()
    # the values each conv read and wrote: x before the chain (its copy x0), the intermediates, x after
    m_outs = dict(zip(io["mids"] + [io["x"], io["x0"]], io["outs"]))
    x_before = vals[m_outs[io["x0"]]]
    after = {t: vals[m_outs[t]] for t in io["mids"] + [io["x"]]}

    def read_value(t):
        return x_before if t in (io["x"], io["x0"]) else after[t]

    worst, fails = 0.0, []
    if kind.startswith("block"):       # the whole block, its bf16 intermediate modelled by block_bound
        (d1, w1, b1), (d2, w2, b2) = convs
        t = lambda a, n: torch.from_numpy(a.reshape(n)).cuda().double()
        Cc = d1.cin
        v, bnd = block_bound(x_before.double(), t(w1, (Cc, Cc, 3, 3)), t(b1, (Cc,)), t(w2, (Cc, Cc, 3, 3)), t(b2, (Cc,)))
        r, over = excess(after[io["x"]], v, bnd)
        net.destroy()
        return lines, r, [f"block: {over} elements over the bound (worst ratio {r:.3g})"] if over else []
    for d, w, b in convs:
        k = int(round(math.sqrt(w.size // (d.cout * d.cin))))
        wt = torch.from_numpy(w.reshape(d.cout, d.cin, k, k)).cuda().double()
        bt = None if b is None else torch.from_numpy(b).cuda().double()
        res = None if d.res < 0 else read_value(d.res).double()
        v, bnd = conv_bound(read_value(d.in_).double(), wt, bt, relu=bool(d.relu), res=res)
        r, over = excess(after[d.out], v, bnd)
        worst = max(worst, r)
        if over:
            fails.append(f"conv t{d.in_}->t{d.out}: {over} elements over the bound (worst ratio {r:.3g})")
    net.destroy()
    return lines, worst, fails


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["block", "block32", "bottleneck", "conv"])
def test_inplace_chains(kind):
    """an in-place BasicBlock (64 channels, or 32 pixel-pair foldable ones) or Bottleneck, whose last conv writes back
    into the block's input slice, its residual, runs unfused and equals float64; so does a single 3x3 conv whose residual
    is its output slice.  Fused, the in-place Bottleneck raced (about 6000 elements of its conv2 output over the bound, by
    up to 2500 times, measured on an H100); the fused in-place blocks happened to be right in that run."""
    lines, worst, fails = run_inplace(kind)
    assert not any(" block " in l or "tc-bottleneck" in l for l in lines), "in-place chain fused:\n" + "\n".join(lines)
    assert any("wgmma" in l for l in lines)
    assert not fails, f"{kind}: " + "; ".join(fails)
    _say(f"   in-place {kind}: {len(lines)} ops unfused, worst |err|/bound {worst:.3f}")
