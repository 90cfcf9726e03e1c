"""The seeded graph generator of tests/net_graphs.py, without a GPU: every seed's graph keeps the library's validity rules,
the write-before-read and write-once rules and the aliasing rule (net_graphs.check_record), the same seed gives the same
graph, the planted items cover every item once over SEEDS, and the restated tensor-core tiling (net_graphs.tc_nt) agrees
with the B2R_CASE table of conv_tc.cu."""
import os

import numpy as np

from tests import net_graphs as NG

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _calls_key(r):
    out = []
    for kind, rid, args in r["calls"]:
        if kind == "conv":
            d, w, b = args
            out.append((kind, rid, tuple(getattr(d, f) for f, _ in d._fields_), w.tobytes(), None if b is None else b.tobytes()))
        elif kind == "sum":
            s = args[0]
            out.append((kind, rid, s.out, s.base, s.n_terms, tuple(s.term), tuple(s.up), s.relu, tuple(s.term_c_off)))
        elif kind == "const":
            out.append((kind, rid, args[:4], args[4].tobytes()))
        else:
            out.append((kind, rid, args))
    return out


def test_generated_graphs_valid():
    for seed in NG.SEEDS:
        g = NG.generate(seed)
        r = g.record()
        bad = NG.check_record(r)
        assert not bad, f"seed {seed}: {bad[:10]}"
        assert 3 <= g.n_ops <= 60
        assert _calls_key(r) == _calls_key(NG.generate(seed).record()), f"seed {seed} is not deterministic"
        ext_out = [t for t, s in r["tensors"].items() if s["ext"] and t not in g.inputs]
        assert ext_out, f"seed {seed} has no external output"


def test_check_record_rejects():
    """the restated rules catch what the generator must never emit"""
    g = NG.generate(0)
    r = g.record()
    conv = next(i for i, c in enumerate(r["calls"]) if c[0] == "conv" and r["tensors"][c[2][0].in_]["C"] >= 16 and
                not r["tensors"][c[2][0].in_]["ext"])
    kind, op, (d, w, b) = r["calls"][conv]
    for field, value, what in (("out", d.in_, "overlaps"), ("in_c_off", r["tensors"][d.in_]["C"], "input slice")):
        d2 = type(d)()
        for f, _ in d._fields_:
            setattr(d2, f, getattr(d, f))
        setattr(d2, field, value)
        if field == "out":
            d2.out_c_off, d2.cout = d.in_c_off, d.cin
        calls = list(r["calls"])
        calls[conv] = (kind, op, (d2, w, b))
        bad = NG.check_record(dict(r, calls=calls))
        assert any(what in x for x in bad), (field, bad)
    # a channel read before any op writes it
    t = len(r["tensors"])
    tensors = dict(r["tensors"])
    tensors[t] = dict(H=16, W=16, C=8, dt=NG.BF16, nchw=0, ext=0, const=False)
    d3 = NG.ConvDesc(t, 0, d.out, d.out_c_off, -1, 0, 0, 8, d.cout, 1, 1, 0, 1, 0, -1, 0)
    bad = NG.check_record(dict(r, tensors=tensors, calls=r["calls"] + [("conv", 999, (d3, w, b))]))
    assert any("read before written" in x for x in bad) and any("twice" in x for x in bad), bad


def test_items_cover_every_row():
    """every planted item lands in some seed, and the items hold one conv for each reachable B2R_CASE row and epilogue"""
    its = NG.items()
    picked = set()
    for seed in NG.SEEDS:
        picked |= set(NG.planted_items(seed, len(its), len(NG.SEEDS)))
    assert picked == set(range(len(its)))
    rows = NG.b2r_rows(open(os.path.join(ROOT, "romp_b200", "csrc", "conv_tc.cu")).read())
    assert len(rows) == len(set(rows)) == 40
    dead = NG.unreachable_rows(rows)
    # the bf16 3x3 256-channel row at N = 64: 288 KiB of resident weights; the streamed plan takes those convs instead
    assert dead == [(3, 256, 64, 2)], dead
    names = {n for n, _ in its}
    for row in rows:
        if row not in dead:
            for epi in ("direct", "generic"):
                assert f"tc {row} {epi}" in names


def test_planner_restatement():
    """plan_workspace on a hand-made op list: exact-size reuse after the last use, in first-freed order"""
    T = {0: dict(H=4, W=4, C=8, dt=NG.BF16, ext=1, const=False)}
    for t in range(1, 6):
        T[t] = dict(H=4, W=4, C=8 if t != 3 else 16, dt=NG.BF16, ext=0, const=False)
    ops = [dict(reads=[0], writes=[1], lane=0), dict(reads=[1], writes=[2], lane=1), dict(reads=[2], writes=[3], lane=0),
           dict(reads=[3], writes=[4], lane=2), dict(reads=[4, 3], writes=[5], lane=0)]
    total, bufs = NG.plan_workspace(T, ops, 4)
    one = (4 * 4 * 8 * 2 * 4 + 1023) // 1024 * 1024
    two = (4 * 4 * 16 * 2 * 4 + 1023) // 1024 * 1024
    # t1 dies at op 1, so t2 gets a new buffer; t3 (other size) a third; t4 takes t1's buffer, t5 t2's
    assert total == 2 * one + two
    assert [[t for t, _ in b["held"]] for b in bufs] == [[1, 4], [2, 5], [3]]
    assert np.array_equal(sorted(len(b["held"]) for b in bufs), [1, 2, 2])
