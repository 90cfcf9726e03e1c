"""BEV's tracker at its thresholds, ties and capacities: oracle/track_oracle.py's edge sequences against the reference's
own tracker (tests/golden/bev_track_edges.npz, tests/golden/make_golden_bev_track_edges.py), decision for decision, and
negative controls: oracles broken on purpose in one rule each must disagree with the reference's rows somewhere, which
shows that the sequences sit on the edges.  Frames where lapjv's extended problem ties (a cost exactly at a limit, two
optimal matchings) are checked against the documented rule instead: a pair at c == lam is dropped."""
import os

import numpy as np
import pytest

from oracle import track_oracle as TO

HERE = os.path.dirname(os.path.abspath(__file__))
KINDS = ["scores", "match", "tie_limit", "tie_limit600", "kalman", "dup", "lifecycle", "ties", "largest", "assign128",
         "assign_tie", "rows126"]
KEYS = ["smpl_thetas", "smpl_betas", "cam", "cam_trans", "params_pred", "center_confs", "pred_batch_ids"]


@pytest.fixture(scope="module")
def golden():
    return np.load(os.path.join(HERE, "golden", "bev_track_edges.npz"))


def load_case(z, kind):
    """-> (EdgeVideo, per-frame reference rows [(ids, inds)], tie frames); the inputs checked against the checksum."""
    v = TO.edge_video(kind)
    chk = float(np.sum([f[k].astype(np.float64).sum() for f in v.frames if f for k in KEYS]))
    assert chk == float(z[f"{kind}/checksum"][0]), f"edge_video({kind!r}) changed"
    assert v.ties == z[f"{kind}/ties"].tolist() and (v.broken if v.broken is not None else -1) == int(z[f"{kind}/broken"][0])
    rows, ids, inds, r0 = z[f"{kind}/rows"], z[f"{kind}/ids"], z[f"{kind}/inds"], 0
    ref = []
    for n in rows.tolist():
        ref.append((ids[r0:r0 + n].tolist(), inds[r0:r0 + n].tolist()))
        r0 += n
    assert r0 == len(ids) and len(ref) == len(v.frames)
    return v, ref


def oracle_rows(v, wrong=()):
    """-> (per-frame (ids, inds), TemporalBEV) of the oracle run on the sequence."""
    sm = TO.TemporalBEV(show_largest=v.show_largest, wrong=wrong)
    out = []
    for f in v.frames:
        o = sm(f, 0) if f else None
        if o is None:
            out.append(([], []))
        elif v.show_largest:
            out.append(([0], o["largest"].tolist()))
        else:
            out.append((o["track_ids"].tolist(), o["det_inds"].tolist()))
    return out, sm


def expected_rows(z, kind):
    """The reference's rows, and on its tie frames the rows of the documented rule (checked on its own below)."""
    v, ref = load_case(z, kind)
    mine, _ = oracle_rows(v)
    return v, [mine[t] if t in v.ties else r for t, r in enumerate(ref)]


@pytest.mark.parametrize("kind", KINDS)
def test_oracle_matches_reference_on_edges(golden, kind):
    z = golden
    v, ref = load_case(z, kind)
    got, sm = oracle_rows(v)
    for t, (g, r) in enumerate(zip(got, ref)):
        if t not in v.ties:
            assert g == r, f"{kind} frame {t}: oracle {g}, reference {r}"
    if v.show_largest:
        return
    tr, l0, frame = sm.tracker, 0, 0
    sm2 = TO.TemporalBEV()                                  # again, frame by frame, for the lists and the filter
    for t, f in enumerate(v.frames):
        if f:
            sm2(f, 0)
        if any(u <= t for u in v.ties):
            break
        tr = sm2.tracker
        assert tr.frame_id == z[f"{kind}/frame_id"][t]
        nt, nl = int(z[f"{kind}/n_tracked"][t]), int(z[f"{kind}/n_lost"][t])
        t_ids, l_ids, st = tr.state()
        lst = t_ids + l_ids
        assert (len(t_ids), len(l_ids)) == (nt, nl), f"{kind} frame {t}"
        np.testing.assert_array_equal(lst, z[f"{kind}/list_ids"][l0:l0 + nt + nl], err_msg=f"{kind} frame {t}")
        np.testing.assert_array_equal([st[i][0] for i in lst], z[f"{kind}/list_state"][l0:l0 + nt + nl])
        np.testing.assert_array_equal([st[i][1] for i in lst], z[f"{kind}/list_act"][l0:l0 + nt + nl])
        mean = np.array([st[i][2] for i in lst]).reshape(-1, 8)
        S = np.array([st[i][3][[0, 0, 4], [0, 4, 4]] for i in lst]).reshape(-1, 3)
        for g, r in ((mean, z[f"{kind}/mean"][l0:l0 + nt + nl]), (S, z[f"{kind}/cov"][l0:l0 + nt + nl])):
            # the reference predicts a pool of fresh tracks with Q rounded to fp32 (their means are fp32)
            rel = np.abs(g - r).max(1) / np.abs(r).max(1) if len(r) else np.zeros(0)
            assert (rel < 1e-6).all(), f"{kind} frame {t}: {rel.max():.2e}"
        l0 += nt + nl
        frame += 1
    margins = {k: sm.tracker.min_margin(k) for k in ("score", "match", "dup", "nearest")}
    print(f"{kind}: {len(v.frames)} frames, relative margins to the thresholds " +
          ", ".join(f"{k} {m:.1e}" for k, m in margins.items()))


def test_tie_frames_follow_the_documented_rule(golden):
    """c == lam drops the pair (300 and 900 on one frame, 600 with a low-score detection); two equal-cost matchings
    both give every track a row."""
    v, ref = load_case(golden, "tie_limit")
    got, _ = oracle_rows(v)
    assert got[2][0] == [2]                                  # anchors 0 (300) and 2 (900, unconfirmed) dropped
    v, _ = load_case(golden, "tie_limit600")
    got, _ = oracle_rows(v)
    assert got[2][0] == [1]                                  # anchor 1's track (600 in the second matching) dropped
    v, _ = load_case(golden, "assign_tie")
    got, _ = oracle_rows(v)
    assert sorted(got[1][0]) == [1, 2, 3] and sorted(got[1][1][:2]) == [0, 1]


@pytest.mark.parametrize("wrong", TO.WRONG)
def test_negative_control_is_rejected(golden, wrong):
    """An oracle with one rule broken disagrees with the reference's rows (the documented rule on tie frames)."""
    where = []
    for kind in KINDS:
        v, exp = expected_rows(golden, kind)
        got, _ = oracle_rows(v, (wrong,))
        where += [(kind, t) for t, (g, e) in enumerate(zip(got, exp)) if g != e]
    print(f"{wrong}: disagrees on {len(where)} frames, first {where[:3]}")
    assert where, f"no edge sequence decides {wrong}"


def test_edge_coverage(golden):
    """Every edge case is in the fixture, and each still holds what it is there for."""
    assert sorted(KINDS) == sorted(TO.EDGE_KINDS)
    for kind in KINDS:
        assert f"{kind}/checksum" in golden, kind
    rows = lambda k: golden[f"{k}/rows"]
    scores = TO.edge_video("scores").frames
    s0 = scores[0]["center_confs"]
    for s in (TO.DET_THRESH, TO.LOW_THRESH):
        assert {s, TO.up(s), TO.down(s)} <= set(s0.tolist())
    v, _ = load_case(golden, "assign128")
    pool = int(golden["assign128/n_tracked"][-2] + golden["assign128/n_lost"][-2])
    assert v.frames[-1]["cam"].shape[0] == 64 and pool == 128                  # the first matching is 128 x 64
    assert rows("assign128")[-1] == 64
    assert rows("rows126").max() == 126 and int(golden["rows126/broken"][0]) == 6
    v, _ = load_case(golden, "rows126")
    assert int(golden["rows126/n_tracked"][5] + golden["rows126/n_lost"][5]) == 128    # full before the broken frame
    v, _ = load_case(golden, "kalman")
    assert v.tracker.frame_id >= 80
    v, _ = load_case(golden, "lifecycle")
    ev = v.tracker.events
    assert ev["refind"] >= 2 and ev["refind_removed"] >= 1 and ev["aged"] >= 2 and ev["lost_in_removed"] >= 1, ev
    assert sum(1 for f in v.frames if not f) >= 5             # frames with nobody, not stepping the tracker
    assert [int(golden[f"{k}/ties"].size) for k in ("tie_limit", "tie_limit600", "assign_tie")] == [1, 1, 1]
    largest = TO.edge_video("largest").frames
    assert any(np.sum(f["cam"][:, 0] == f["cam"][:, 0].max()) > 1 for f in largest)
