"""BEV's tracker step (csrc/track.cu, b200romp_bev_track_step) at its thresholds, ties and capacities: every edge
sequence of oracle/track_oracle.py against the reference's own tracker (tests/golden/bev_track_edges.npz).

* Row counts, track ids and detection indices equal the reference's exactly at batch sizes 1, 7 and 64, and the batch
  sizes agree bit for bit.  On frames where lapjv ties the documented rule decides: a pair at c == lam is dropped; with
  two optimal matchings, any optimal one.  A full 128-entry table sets the broken status on the frame the fixture names.
* The smoothed pose, betas and cam against the fp64 One-Euro recurrence with the running first-order bound of
  test_gpu_romp_post_fp64.py; cam_trans is bev/post_parser.py's fp32 formula of the smoothed cam, exactly.
* The 128 x 64 first matching and the equal-cost one: the total fp64 cost of the kernel's matching (read off its rows:
  the filter gain is near 1 there, so each row's nearest detection is its matched one) equals scipy's optimum of the
  extended problem.
* Interleaved as streams of one streams handle, every sequence equals its solo run bit for bit, including the frame whose
  126 rows nearly fill its 2 x 64 window and the stream whose table fills.
Each case prints its relative margins to the thresholds."""
import numpy as np
import pytest

from oracle import track_oracle as TO
from tests.test_gpu_bev_temporal import Stage
from tests.test_gpu_romp_post_fp64 import OneEuro64, check_one_euro
from tests.test_gpu_video_streams import StreamStage, interleave, same
from tests.test_oracle_bev_track_edges import KINDS, expected_rows, golden  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu


def run(v, batch, upto=None):
    """The sequence through a default handle in batches; -> (per-frame rows or None, statuses)."""
    frames = v.frames[:upto]
    st, out, statuses = Stage(show_largest=v.show_largest), [], []
    for c0 in range(0, len(frames), batch):
        r, status = st.step(frames[c0:c0 + batch], [0] * len(frames[c0:c0 + batch]))
        out += r
        statuses.append(status)
    return out, statuses


def rows_of(r):
    return ([], []) if r is None else (r["ids"].tolist(), r["det"].tolist())


def pool_costs(v, t):
    """(pool track ids, fp64 cost matrix pool x detections) of stepped frame t's first matching, from the oracle run
    on the frames before it."""
    sm = TO.TemporalBEV()
    for f in v.frames[:t]:
        if f:
            sm(f, 0)
    tr = sm.tracker
    pool = [x for x in tr.tracked if x.activated] + [x for x in tr.lost if x.id not in {y.id for y in tr.tracked}]
    pts = TO.tracking_points(v.frames[t]["cam"], v.frames[t]["cam_trans"]).astype(np.float64)
    return [x.id for x in pool], np.linalg.norm(np.array([TO.predicted(x)[:4] for x in pool])[:, None] - pts[None], axis=2)


def matching_value(ids, cost, rows, lam=TO.MATCH):
    """Extended-problem value of the matching given by rows (track id, detection) restricted to the pool."""
    pos = {i: k for k, i in enumerate(ids)}
    pairs = [(pos[i], d) for i, d in zip(*rows) if i in pos]
    assert len({d for _, d in pairs}) == len(pairs), "two pool tracks on one detection"
    n, m = cost.shape
    return sum(cost[i, j] for i, j in pairs) + (n - len(pairs) + m - len(pairs)) * lam / 2


@pytest.mark.parametrize("kind", KINDS)
def test_track_step_edges_equal_reference(golden, kind):
    v, exp = expected_rows(golden, kind)
    broken = v.broken
    upto = None if broken is None else broken + 1
    runs = {}
    for batch in (1, 7, 64):
        got, statuses = run(v, batch, upto)
        if broken is None:
            assert all(s[0] == 0 for s in statuses), statuses
        else:                                                # the table fills on that frame, not before
            assert statuses[-1][0] == 1 and all(s[0] == 0 for s in statuses[:-1]), statuses
            got = got[:broken]
        for t, r in enumerate(got):
            g = rows_of(r)
            if kind == "assign_tie" and t in v.ties:         # any of the optimal matchings
                assert sorted(g[0]) == sorted(exp[t][0]), (kind, t, g, exp[t])
            else:
                assert g == exp[t], f"{kind} batch {batch} frame {t}: kernel {g}, expected {exp[t]}"
        runs[batch] = got
    for b in (7, 64):
        for t, (x, y) in enumerate(zip(runs[1], runs[b])):
            same(x, y, f"{kind} frame {t}, batch 1 vs {b}")
    # smoothed values: the fp64 recurrence and its bound, on the kernel's rows
    got, worst = runs[1], {}
    oe = OneEuro64(2 * 256, 3.0, not v.show_largest, n_betas=11)
    for t, r in enumerate(got):
        if r is None:
            continue
        f = v.frames[t]
        d = r["det"]
        slots = np.zeros(1, int) if v.show_largest else r["ids"].astype(int)
        y, b_y = oe.step(slots, f["smpl_thetas"][d].astype(np.float64), f["smpl_betas"][d].astype(np.float64),
                         f["cam"][d].astype(np.float64))
        check_one_euro("", oe, y, b_y, r["thetas"], r["betas"], r["cam"], worst)
        np.testing.assert_array_equal(r["cam_trans"], TO.cam_to_trans(r["cam"]))
        np.testing.assert_array_equal(r["params"], f["params_pred"][d])
        np.testing.assert_array_equal(r["conf"], f["center_confs"][d])
    assert all(w <= 1.0 for w in worst.values()), worst
    if not v.show_largest:
        tr = TO.TemporalBEV()
        for f in v.frames[:upto]:
            if f:
                tr(f, 0)
        marg = ", ".join(f"{k} {tr.tracker.min_margin(k):.1e}" for k in ("score", "match", "dup", "nearest"))
    else:
        c = [np.sort(f["cam"][:, 0])[::-1] for f in v.frames if f]
        marg = "largest " + f"{min(float(x[0] - x[1]) for x in c if len(x) > 1):.1e}"
    print(f"{kind}: {len(got)} frames, worst err/bound " + ", ".join(f"{k} {w:.2f}" for k, w in worst.items()) +
          f"; relative margins {marg}")


@pytest.mark.parametrize("kind", ["assign128", "assign_tie"])
def test_track_step_matching_is_optimal(golden, kind):
    v, exp = expected_rows(golden, kind)
    t = len(v.frames) - 1
    ids, cost = pool_costs(v, t)
    best, ua, ub = TO.lap_extended(cost, TO.MATCH)
    opt = sum(cost[i, j] for i, j in best) + (len(ua) + len(ub)) * TO.MATCH / 2
    if kind == "assign128":
        assert cost.shape == (128, 64)
        assert sorted((ids[i], j) for i, j in best) == sorted(zip(*exp[t])), "rows do not show the matching"
        assert TO.assignment_margin(cost, TO.MATCH) > 1e-3
    got, _ = run(v, 64)
    val = matching_value(ids, cost, rows_of(got[t]))
    print(f"{kind}: {cost.shape[0]} x {cost.shape[1]}, kernel {val:.9f}, optimum {opt:.9f}")
    assert abs(val - opt) <= 1e-9 * opt


@pytest.mark.parametrize("mode,batch", [("round", 64), ("burst", 7)])
def test_track_step_edges_as_streams(mode, batch):
    """Every tracked edge sequence as one stream; each equals its solo run bit for bit."""
    vs = [TO.edge_video(k) for k in KINDS if not TO.EDGE_KINDS[k][1]]
    seqs = [v.frames for v in vs]
    order = interleave([len(s) for s in seqs], mode, seed=1)
    st = StreamStage(len(seqs))
    got = [[None] * len(s) for s in seqs]
    failed = set()
    for c0 in range(0, len(order), batch):
        ch = order[c0:c0 + batch]
        r, status = st.step([seqs[k][t] for k, t in ch], [k for k, _ in ch])
        for (k, t), x, s in zip(ch, r, status[2:]):
            got[k][t] = x
            if s < 0:
                failed.add((k, t))
    for k, v in enumerate(vs):
        solo, _ = run(v, 1, None if v.broken is None else v.broken + 1)
        n = len(v.frames) if v.broken is None else v.broken
        assert {t for kk, t in failed if kk == k} == set(range(n, len(v.frames))), k
        for t in range(n):
            same(got[k][t], solo[t], f"stream {k} frame {t}")
        print(f"stream {k}: {n} frames equal the solo run" + ("" if v.broken is None else ", then the full table fails it"))
