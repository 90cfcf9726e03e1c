"""BEV video mode: oracle/track_oracle.py against the reference's own tracker and BEV.temporal_optimization
(tests/golden/bev_track.npz), the kron(S, I4) covariance structure the device kernel relies on, and the c - lam
matching against brute force on the extended assignment problem."""
import os

import numpy as np
import pytest

from oracle import track_oracle as TO

HERE = os.path.dirname(os.path.abspath(__file__))
CASES = ["walk0", "walk1", "walk2", "signals", "largest", "gaps"]
KEYS = ["smpl_thetas", "smpl_betas", "cam", "cam_trans", "params_pred", "center_confs", "pred_batch_ids"]


@pytest.fixture(scope="module")
def golden():
    return np.load(os.path.join(HERE, "golden", "bev_track.npz"))


def _inputs(z, name):
    seed, frames, p0, p1, empty_every, largest, two, kind = z[f"{name}/case"].tolist()
    seq = TO.make_video(kind, seed, frames, (p0, p1), empty_every=empty_every)
    chk = float(np.sum([f[k].astype(np.float64).sum() for f in seq if f for k in KEYS]))
    assert chk == pytest.approx(float(z[f"{name}/checksum"][0]), rel=1e-12), "synthetic_video changed"
    return seq, bool(largest)


@pytest.mark.parametrize("name", CASES)
def test_oracle_matches_reference_tracker(golden, name):
    z = golden
    seq, largest = _inputs(z, name)
    sm = TO.TemporalBEV(show_largest=largest)
    sig, rows = z[f"{name}/sig"], z[f"{name}/rows"]
    ids, inds = z[f"{name}/ids"], z[f"{name}/inds"]
    r0 = s0 = l0 = k0 = 0
    smooth_frames = 40
    for t, f in enumerate(seq):
        out = sm(f, int(sig[t])) if f else None
        n = 0 if out is None else len(out["cam"])
        assert n == rows[t], f"frame {t}: {n} rows, reference {rows[t]}"
        if n:
            if largest:
                assert out["largest"][0] == inds[r0]
            else:
                np.testing.assert_array_equal(out["track_ids"], ids[r0:r0 + n], err_msg=f"frame {t}")
                np.testing.assert_array_equal(out["det_inds"], inds[r0:r0 + n], err_msg=f"frame {t}")
            if t < smooth_frames:
                for k, g in (("smpl_thetas", "thetas"), ("smpl_betas", "betas"), ("cam", "cam"), ("cam_trans", "cam_trans")):
                    np.testing.assert_allclose(out[k], z[f"{name}/{g}"][s0:s0 + n], atol=1e-6, rtol=1e-6, err_msg=f"frame {t} {k}")
                s0 += n
            r0 += n
        if largest:
            continue
        tr = sm.tracker
        assert tr.frame_id == z[f"{name}/frame_id"][t]
        nt, nl = int(z[f"{name}/n_tracked"][t]), int(z[f"{name}/n_lost"][t])
        t_ids, l_ids, st = tr.state()
        lst = t_ids + l_ids
        assert (len(t_ids), len(l_ids)) == (nt, nl), f"frame {t}"
        np.testing.assert_array_equal(lst, z[f"{name}/list_ids"][l0:l0 + nt + nl], err_msg=f"frame {t}")
        np.testing.assert_array_equal([st[i][0] for i in lst], z[f"{name}/list_state"][l0:l0 + nt + nl])
        np.testing.assert_array_equal([st[i][1] for i in lst], z[f"{name}/list_act"][l0:l0 + nt + nl])
        if t < 60 or t % 10 == 0:
            mean = np.array([st[i][2] for i in lst]).reshape(-1, 8)
            S = np.array([st[i][3][[0, 0, 4], [0, 4, 4]] for i in lst]).reshape(-1, 3)
            for got, ref in ((mean, z[f"{name}/mean"][k0:k0 + nt + nl]), (S, z[f"{name}/cov"][k0:k0 + nt + nl])):
                # relative to each track's largest entry: the reference starts P in fp32 (kalman_filter_3dcenter.py:76-85)
                rel = np.abs(got - ref).max(1) / np.abs(ref).max(1) if len(ref) else np.zeros(0)
                assert (rel < 1e-6).all(), f"frame {t}: {rel.max():.2e}"
            k0 += nt + nl
        l0 += nt + nl
    assert r0 == len(ids)
    if not largest:
        assert tr.min_margin() > 1e-6, "a decision came near its threshold"
    if name == "gaps":
        # every lifecycle path of the tracker, seen in the reference's own lists ...
        lists, seen = [], 0
        for t in range(len(seq)):
            n = int(z[f"{name}/n_tracked"][t] + z[f"{name}/n_lost"][t])
            nt = int(z[f"{name}/n_tracked"][t])
            li, ls, la = (z[f"{name}/{k}"][seen:seen + n] for k in ("list_ids", "list_state", "list_act"))
            lists.append((set(li[:nt].tolist()), set(li[nt:].tolist()), dict(zip(li.tolist(), ls.tolist())),
                          {i for i, a in zip(li.tolist(), la.tolist()) if not a}))
            seen += n
        aged = sum(any(st == TO.REMOVED for st in l[2].values()) for l in lists)
        refound = sum(len(lists[t - 1][1] & lists[t][0]) for t in range(1, len(lists)))
        unconfirmed_gone = sum(len(lists[t - 1][3] - lists[t][0] - lists[t][1]) for t in range(1, len(lists)))
        assert aged >= 2 and refound >= 2 and unconfirmed_gone >= 2, (aged, refound, unconfirmed_gone)
        # ... and in the oracle's
        ev = tr.events
        assert ev["aged"] >= 2 and ev["refind"] >= 1 and ev["refind_removed"] >= 1 and ev["unconfirmed_removed"] >= 2, ev
        assert ev["lost_in_removed"] >= 1, ev
    elif not largest:
        assert len(set(ids.tolist())) > 10                   # the random walks exercise crowds and crossings


def test_covariance_is_kron_s_i4(golden):
    """The reference's own covariances: P = kron(S, I4), S a symmetric 2x2 (the device keeps 3 scalars per track)."""
    worst = 0.0
    for name in [c for c in CASES if c != "largest"]:
        P = golden[f"{name}/covfull"]
        assert len(P) > 50
        for p in P:
            S = p[[0, 0, 4, 4], [0, 4, 0, 4]].reshape(2, 2)
            worst = max(worst, np.abs(p - np.kron(S, np.eye(4))).max() / np.abs(p).max())
    assert worst < 1e-12, worst


def test_oracle_covariance_matches_closed_form():
    """The kernel's 3-scalar recursion (predict: a+2b+c+q_p, b+c, c+q_v; update: gain a/S, b/S) equals the oracle's
    8x8 matrices on a random sequence of predicts and updates."""
    rs = np.random.RandomState(0)
    z = rs.uniform(10, 200, 4)
    m, P = TO.kf_initiate(z)
    a, b, c = P[0, 0], 0.0, P[4, 4]
    for _ in range(50):
        h = m[3]
        m, P = TO.kf_predict(m, P)
        a, b, c = a + 2 * b + c + (h / 20) ** 2, b + c, c + (h / 160) ** 2
        if rs.rand() < 0.7:
            r = (m[3] / 20) ** 2
            s = a + r
            m, P = TO.kf_update(m, P, m[:4] + rs.normal(0, 3, 4))
            a, b, c = a - a * a / s, b - a * b / s, c - b * b / s
        np.testing.assert_allclose(P[[0, 0, 4], [0, 4, 4]], [a, b, c], rtol=1e-9)


@pytest.mark.parametrize("seed", range(40))
def test_margin_matching_equals_brute_force(seed):
    rs = np.random.RandomState(seed)
    n, m = rs.randint(1, 6), rs.randint(1, 6)
    lam = 300.0
    cost = rs.uniform(0, 2 * lam, (n, m))
    best = TO.brute_force_extended(cost, lam)
    for solve in (TO.lap_extended, TO.lap_margin):
        matches, ua, ub = solve(cost, lam)
        val = sum(cost[i, j] for i, j in matches) + (len(ua) + len(ub)) * lam / 2.0
        assert val == pytest.approx(best, rel=1e-12, abs=1e-9), solve.__name__
        assert sorted(ua + [i for i, _ in matches]) == list(range(n))
        assert sorted(ub + [j for _, j in matches]) == list(range(m))
    assert TO.lap_extended(cost, lam)[0] == TO.lap_margin(cost, lam)[0]    # continuous costs: the optimum is unique
