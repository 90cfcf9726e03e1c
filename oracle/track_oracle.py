"""CPU oracle of BEV's video mode (``-t/--temporal_optimize``).  TEST INFRASTRUCTURE ONLY.

Restates the reference's 3-D-centre ByteTrack (simple_romp/tracker/byte_tracker_3dcenter.py, kalman_filter_3dcenter.py,
matching.py) and ``BEV.temporal_optimization`` (bev/main.py:260-287), reusing oracle/temporal_oracle.py's One-Euro.
The assignment ``lap.lapjv(cost, extend_cost=True, cost_limit=lam)`` (matching.py:38-49) is solved with scipy's
``linear_sum_assignment`` on the same extended (n+m)x(n+m) matrix.  Every threshold decision records how far it
cleared its threshold (``Tracker.margins``) so tests can reject sequences that come near a tie.  Pinned by
tests/test_oracle_bev_track_golden.py against tests/golden/bev_track.npz (outputs of the reference's own tracker).
"""
import collections
import itertools

import numpy as np
from scipy.optimize import linear_sum_assignment

from . import temporal_oracle as T

F = np.float32
NEW, TRACKED, LOST, REMOVED = 0, 1, 2, 3          # basetrack.TrackState
DET_THRESH, LOW_THRESH = F(0.12), F(0.05)         # bev/main.py:121, compared in fp32
MATCH, MAX_LOST, DUP = 300.0, 60, 60.0
STD_POS, STD_VEL = 1.0 / 20, 1.0 / 160
TAN_FOV = np.float32(np.tan(np.radians(30.0)))


# ----------------------------------------------------------------------------------------------------------------
# assignment
def lap_extended(cost, lam, keep_equal=False):
    """lap.lapjv(cost, extend_cost=True, cost_limit=lam) as linear_assignment uses it: the (n+m)^2 problem with the
    cost in the top-left block, lam/2 in both off-diagonal blocks and 0 in the dummy block.  Returns (matches [(i, j)],
    unmatched rows ascending, unmatched columns ascending).  A pair at exactly c = lam ties with leaving both unmatched
    (lam/2 + lam/2); such a pair is dropped, the rule romp_b200/csrc/track.cu documents (keep_equal: kept instead)."""
    n, m = cost.shape
    if n == 0 or m == 0:
        return [], list(range(n)), list(range(m))
    ext = np.full((n + m, n + m), lam / 2.0)
    ext[:n, :m] = np.where(cost == lam, np.nextafter(lam, 0.0), cost) if keep_equal else cost
    ext[n:, m:] = 0.0
    r, c = linear_sum_assignment(ext)
    x = np.full(n, -1)
    y = np.full(m, -1)
    for i, j in zip(r, c):
        if i < n and j < m and (cost[i, j] < lam or keep_equal):
            x[i], y[j] = j, i
    return [(i, int(x[i])) for i in range(n) if x[i] >= 0], [i for i in range(n) if x[i] < 0], [j for j in range(m) if y[j] < 0]


def lap_margin(cost, lam):
    """The same problem as a minimum-cost (not necessarily perfect) matching with edge costs c - lam: the Hungarian
    method (shortest augmenting paths with potentials) on the k x k matrix min(c - lam, 0), k = max(n, m), zero padded,
    keeping the pairs with c - lam < 0.  The algorithm romp_b200/csrc/track.cu runs."""
    n, m = cost.shape
    if n == 0 or m == 0:
        return [], list(range(n)), list(range(m))
    k = max(n, m)
    a = np.zeros((k + 1, k + 1))
    a[1:n + 1, 1:m + 1] = np.minimum(cost - lam, 0.0)
    u, v, p, way = np.zeros(k + 1), np.zeros(k + 1), np.zeros(k + 1, int), np.zeros(k + 1, int)
    for i in range(1, k + 1):
        p[0], j0 = i, 0
        minv, used = np.full(k + 1, np.inf), np.zeros(k + 1, bool)
        while True:
            used[j0] = True
            i0, delta, j1 = p[j0], np.inf, 0
            for j in range(1, k + 1):
                if not used[j]:
                    cur = a[i0, j] - u[i0] - v[j]
                    if cur < minv[j]:
                        minv[j], way[j] = cur, j0
                    if minv[j] < delta:
                        delta, j1 = minv[j], j
            for j in range(k + 1):
                if used[j]:
                    u[p[j]] += delta
                    v[j] -= delta
                else:
                    minv[j] -= delta
            j0 = j1
            if p[j0] == 0:
                break
        while j0:
            j1 = way[j0]
            p[j0] = p[j1]
            j0 = j1
    x = np.full(n, -1)
    y = np.full(m, -1)
    for j in range(1, m + 1):
        i = p[j] - 1
        if i < n and cost[i, j - 1] - lam < 0:
            x[i], y[j - 1] = j - 1, i
    return [(i, int(x[i])) for i in range(n) if x[i] >= 0], [i for i in range(n) if x[i] < 0], [j for j in range(m) if y[j] < 0]


def brute_force_extended(cost, lam):
    """Optimal value of the extended problem by enumerating every (partial) matching.  Small n, m only."""
    n, m = cost.shape
    best = n * lam / 2.0 + m * lam / 2.0
    for r in range(1, min(n, m) + 1):
        for rows in itertools.combinations(range(n), r):
            for cols in itertools.permutations(range(m), r):
                v = sum(cost[i, j] for i, j in zip(rows, cols)) + (n - r) * lam / 2.0 + (m - r) * lam / 2.0
                best = min(best, v)
    return best


# ----------------------------------------------------------------------------------------------------------------
# Kalman filter (kalman_filter_3dcenter.py), full 8x8 matrices like the reference
_Fm = np.eye(8)
_Fm[:4, 4:] = np.eye(4)
_H = np.eye(4, 8)


def kf_initiate(z):
    """The reference's initial covariance is fp32 (a float32 measurement scales the standard deviations)."""
    h = F(z[3])
    sp, sv = F(2 * STD_POS) * h, F(10 * STD_VEL) * h
    return np.r_[np.asarray(z, np.float64), np.zeros(4)], np.diag(np.r_[[sp * sp] * 4, [sv * sv] * 4].astype(F).astype(np.float64))


def kf_predict(mean, P, q_vel=True):
    """q_vel=False leaves out the h/160 velocity noise (a wrong filter, for negative controls)."""
    h = mean[3]
    q = np.r_[[STD_POS * h] * 4, [STD_VEL * h if q_vel else 0.0] * 4]
    return _Fm @ mean, _Fm @ P @ _Fm.T + np.diag(q * q)


def kf_update(mean, P, z):
    r = STD_POS * mean[3]
    S = _H @ P @ _H.T + np.diag([r * r] * 4)
    K = np.linalg.solve(S, (P @ _H.T).T).T
    return mean + (np.asarray(z, np.float64) - _H @ mean) @ K.T, P - K @ S @ K.T


# ----------------------------------------------------------------------------------------------------------------
class Track:
    def __init__(self, z, score):
        self.z, self.score = np.asarray(z, F), score
        self.mean = self.P = None
        self.state, self.activated, self.in_removed = NEW, False, False
        self.id = self.frame_id = self.start_frame = 0

    @property
    def point(self):
        return self.z.astype(np.float64) if self.mean is None else self.mean[:4]


def _dist(a, b):
    if len(a) == 0 or len(b) == 0:
        return np.zeros((len(a), len(b)))
    return np.linalg.norm(np.array(a)[:, None] - np.array(b)[None], axis=2)


def _argbest(v, last, arg):
    """arg (np.argmin / np.argmax) of v: the first index on ties, the last one when last."""
    return len(v) - 1 - int(arg(v[::-1])) if last else int(arg(v))


def _joint(a, b):
    ids = {t.id for t in a}
    return a + [t for t in b if t.id not in ids]


def _sub(a, b):
    ids = {t.id for t in b}
    return [t for t in a if t.id not in ids]


WRONG = ("score_le", "match_le", "dup_le", "lost_ge", "no_zero_vel", "no_q_vel", "last_on_ties")


class Tracker:
    """Tracker(det_thresh=0.12, low_conf_det_thresh=0.05, track_buffer=60, match_thresh=300, frame_rate=30), BT:6-147.
    Ids count from 1 per instance.  ``margins`` collects (kind, distance to the threshold) of every decision.
    ``wrong``: rules from WRONG deliberately broken, so tests can show that a sequence decides them: ``<=`` / ``>=``
    in place of the strict score, matching and duplicate compares, removal at ``>= 60`` lost frames, no ``mean[7] = 0``
    for lost tracks, Q without its velocity term, the last nearest detection on ties."""

    def __init__(self, wrong=()):
        assert set(wrong) <= set(WRONG), wrong
        self.wrong = set(wrong)
        self.tracked, self.lost = [], []
        self.frame_id, self.count = 0, 0
        self.margins = []
        self.events = collections.Counter()          # refind, refind_removed, aged, unconfirmed_removed, lost_in_removed

    def _assign(self, tracks, dets, lam):
        c = _dist([t.point for t in tracks], [d.point for d in dets])
        if c.size:
            self.margins.append(("match", float(np.abs(c - lam).min()) / lam))
        return lap_extended(c, lam, keep_equal="match_le" in self.wrong)

    def update(self, points, scores):
        """points fp32 [N,4], scores fp32 [N] -> (track ids, detection index per row)."""
        points, scores = np.asarray(points, F), np.asarray(scores, F)
        self.frame_id += 1
        fid = self.frame_id
        if len(scores):
            self.margins.append(("score", float(min(np.abs(scores - DET_THRESH).min(), np.abs(scores - LOW_THRESH).min()))))
        if "score_le" in self.wrong:
            high, low = scores >= DET_THRESH, (scores >= LOW_THRESH) & (scores < DET_THRESH)
        else:
            high, low = scores > DET_THRESH, (scores > LOW_THRESH) & (scores < DET_THRESH)
        dets = [Track(p, s) for p, s in zip(points[high], scores[high])]
        activated, refind, lost_new, removed_new = [], [], [], []
        unconfirmed = [t for t in self.tracked if not t.activated]
        pool = _joint([t for t in self.tracked if t.activated], self.lost)
        for t in pool:                                                         # STrack.multi_predict
            m = t.mean.copy()
            if t.state != TRACKED and "no_zero_vel" not in self.wrong:
                m[7] = 0
            t.mean, t.P = kf_predict(m, t.P, "no_q_vel" not in self.wrong)

        def upd(t, d, refound):
            t.mean, t.P = kf_update(t.mean, t.P, d.z)
            t.state, t.activated, t.frame_id, t.score = TRACKED, True, fid, d.score
            (refind if refound else activated).append(t)

        matches, u_track, u_det = self._assign(pool, dets, MATCH)
        for it, idt in matches:
            if pool[it].state != TRACKED:
                self.events["refind" if pool[it].state == LOST else "refind_removed"] += 1
            upd(pool[it], dets[idt], pool[it].state != TRACKED)
        dets2 = dets if low.any() else []                                      # BT:75-80: the high-score detections
        r_tracked = [pool[i] for i in u_track if pool[i].state == TRACKED]
        matches, u_track2, _ = self._assign(r_tracked, dets2, MATCH * 2)
        for it, idt in matches:
            upd(r_tracked[it], dets2[idt], False)
        for it in u_track2:
            t = r_tracked[it]
            if t.state != LOST:
                t.state = LOST
                lost_new.append(t)
        rem = [dets[i] for i in u_det]
        matches, u_unc, u_det3 = self._assign(unconfirmed, rem, MATCH * 3)
        for it, idt in matches:
            upd(unconfirmed[it], rem[idt], False)
        for it in u_unc:
            self.events["unconfirmed_removed"] += 1
            unconfirmed[it].state = REMOVED
            removed_new.append(unconfirmed[it])
        for i in u_det3:                                                       # STrack.activate
            t = rem[i]
            self.count += 1
            t.id = self.count
            t.mean, t.P = kf_initiate(t.z)
            t.state, t.activated, t.frame_id, t.start_frame = TRACKED, fid == 1, fid, fid
            activated.append(t)
        for t in self.lost:
            if fid - t.frame_id > MAX_LOST or ("lost_ge" in self.wrong and fid - t.frame_id == MAX_LOST):
                self.events["aged"] += t.state == LOST
                t.state = REMOVED
                removed_new.append(t)
        tracked = [t for t in self.tracked if t.state == TRACKED]
        tracked = _joint(_joint(tracked, activated), refind)
        lost = _sub(self.lost, tracked) + lost_new
        self.events["lost_in_removed"] += sum(t.in_removed for t in lost_new)   # lost again after a removal: dropped
        lost = [t for t in lost if not t.in_removed]                          # sub_stracks(lost, self.removed_stracks)
        for t in removed_new:
            t.in_removed = True
        pd = _dist([t.mean[:2] for t in tracked], [t.mean[:2] for t in lost])  # remove_duplicate_stracks, dim=2
        if pd.size:
            self.margins.append(("dup", float(np.abs(pd - DUP).min()) / DUP))
        dupa, dupb = set(), set()
        for p, q in zip(*np.where(pd <= DUP if "dup_le" in self.wrong else pd < DUP)):
            if tracked[p].frame_id - tracked[p].start_frame > lost[q].frame_id - lost[q].start_frame:
                dupb.add(q)
            else:
                dupa.add(p)
        self.tracked = [t for i, t in enumerate(tracked) if i not in dupa]
        self.lost = [t for i, t in enumerate(lost) if i not in dupb]
        ids, inds = [], []
        for t in self.tracked:                                                 # get_tracked_ids_byte, BT:149-159
            if not t.activated:
                continue
            d = np.linalg.norm(t.mean[:4][None] - points.astype(np.float64), axis=1)
            if len(d) > 1:
                s = np.sort(d)
                self.margins.append(("nearest", float(s[1] - s[0]) / max(float(s[1]), 1e-9)))
            ids.append(t.id)
            inds.append(_argbest(d, "last_on_ties" in self.wrong, np.argmin))
        return ids, inds

    def state(self):
        """(tracked ids, lost ids, {id: (state, activated, mean, P)}) of the listed tracks."""
        return ([t.id for t in self.tracked], [t.id for t in self.lost],
                {t.id: (t.state, t.activated, t.mean.copy(), t.P.copy()) for t in self.tracked + self.lost})

    def min_margin(self, kind=None):
        v = [m for k, m in self.margins if kind is None or k == kind]
        return min(v) if v else np.inf


# ----------------------------------------------------------------------------------------------------------------
def cam_to_trans(cam):
    """denormalize_cam_params_to_trans (bev/post_parser.py:114-128) in fp32."""
    cam = np.asarray(cam, F)
    depth = F(1) / (cam[:, 0] * TAN_FOV + F(1e-3))
    return np.stack([cam[:, 2] * depth * TAN_FOV, cam[:, 1] * depth * TAN_FOV, depth], 1).astype(F)


def tracking_points(cam, cam_trans):
    """bev/main.py:269-272 in fp32 (image_scale 128, depth_scale 30)."""
    cam, cam_trans = np.asarray(cam, F), np.asarray(cam_trans, F)
    return np.concatenate([(cam[:, [2, 1]] + F(1)) * F(128), cam_trans[:, [2]] * F(30), cam[:, [0]] * F(128) / F(2)], 1)


class TemporalBEV:
    """BEV.temporal_optimization (bev/main.py:260-287) with one tracker shared by every signal_ID."""

    def __init__(self, show_largest=False, smooth_coeff=3.0, wrong=()):
        self.show_largest, self.smooth_coeff = show_largest, smooth_coeff
        self.last_on_ties = "last_on_ties" in wrong
        self.tracker = None if show_largest else Tracker(wrong)
        self.filters = {}

    def __call__(self, out, signal_ID=0):
        """out: numpy dict of the result_keys for one frame with at least one detection.  Returns the smoothed dict
        (cam_trans recomputed from the smoothed cam, bev/main.py:169), or None."""
        out = {k: np.array(v) for k, v in out.items()}
        if self.show_largest:
            f = self.filters.setdefault(signal_ID, T.make_filters(self.smooth_coeff))
            k = _argbest(out["cam"][:, 0], self.last_on_ties, np.argmax)
            th, be, ca = T.smooth(f, out["smpl_thetas"][k], out["smpl_betas"][k], out["cam"][k])
            out["smpl_thetas"], out["smpl_betas"], out["cam"] = th[None], be[None], ca[None]
            out["largest"] = np.array([k])
        else:
            pts = tracking_points(out["cam"], out["cam_trans"])
            ids, inds = self.tracker.update(pts, out["center_confs"])
            if not ids:
                return None
            out = {k: v[inds] for k, v in out.items()}
            fs = self.filters.setdefault(signal_ID, {})
            for r, tid in enumerate(ids):
                f = fs.setdefault(tid, T.make_filters(self.smooth_coeff))
                out["smpl_thetas"][r], out["smpl_betas"][r], out["cam"][r] = T.smooth(
                    f, out["smpl_thetas"][r], out["smpl_betas"][r], out["cam"][r])
            out["track_ids"] = np.array(ids, np.int32)
            out["det_inds"] = np.array(inds, np.int64)
        out["cam_trans"] = cam_to_trans(out["cam"])
        return out


# ----------------------------------------------------------------------------------------------------------------
def synthetic_video(seed, frames=200, people=(6, 12), max_dets=64, low_frac=0.08, empty_every=0):
    """Seeded random walks of people's cams with births, occlusion gaps (short and longer than 60 frames), detections
    with scores in (0.05, 0.12) and crossing paths.  Returns a list of per-frame numpy dicts with the result_keys
    (thetas/betas/params random per person, varying slowly) - frames with nobody are empty dicts."""
    rs = np.random.RandomState(seed)
    n_max = int(rs.randint(people[0], people[1] + 1))
    P = []
    for p in range(n_max):
        birth = int(rs.randint(0, frames // 2)) if p >= people[0] else 0
        gaps = []
        for _ in range(rs.randint(0, 3)):
            g0 = int(rs.randint(birth + 1, frames))
            gaps.append((g0, g0 + int(rs.choice([rs.randint(2, 20), rs.randint(62, 90)]))))
        P.append(dict(birth=birth, gaps=gaps, cam=np.array([rs.uniform(0.25, 0.6), rs.uniform(-0.8, 0.8), rs.uniform(-0.8, 0.8)]),
                      vel=np.array([0.0, rs.normal(0, 0.01), rs.normal(0, 0.012)]),
                      th=rs.normal(0, 0.3, 72), be=rs.normal(0, 0.4, 11), pp=rs.normal(0, 1, 146)))
    seq = []
    for t in range(frames):
        rows = []
        if not (empty_every and t % empty_every == empty_every - 1):
            for p in P:
                p["cam"] = p["cam"] + p["vel"] + np.r_[rs.normal(0, 0.004), rs.normal(0, 0.002, 2)]
                p["cam"][0] = np.clip(p["cam"][0], 0.15, 0.8)
                for a in (1, 2):
                    if abs(p["cam"][a]) > 0.95:
                        p["vel"][a] = -p["vel"][a]
                if t < p["birth"] or any(g0 <= t < g1 for g0, g1 in p["gaps"]):
                    continue
                s = rs.uniform(0.06, 0.115) if rs.rand() < low_frac else rs.uniform(0.13, 0.9)
                p["th"] += rs.normal(0, 0.02, 72)
                p["be"] += rs.normal(0, 0.01, 11)
                rows.append((p["cam"].copy(), s, p["th"].copy(), p["be"].copy(), p["pp"] + rs.normal(0, 0.01, 146)))
        rows = rows[:max_dets]
        if not rows:
            seq.append({})
            continue
        order = rs.permutation(len(rows))                                  # the parse order is not the person order
        cam = np.array([rows[i][0] for i in order], F)
        seq.append(dict(cam=cam, cam_trans=cam_to_trans(cam), center_confs=np.array([rows[i][1] for i in order], F),
                        smpl_thetas=np.array([rows[i][2] for i in order], F), smpl_betas=np.array([rows[i][3] for i in order], F),
                        params_pred=np.array([rows[i][4] for i in order], F), pred_batch_ids=np.zeros(len(rows), np.int64)))
    return seq


def _frame_dict(rows, rs):
    order = rs.permutation(len(rows))                                  # the parse order is not the person order
    cam = np.array([rows[i][0] for i in order], F)
    return dict(cam=cam, cam_trans=cam_to_trans(cam), center_confs=np.array([rows[i][1] for i in order], F),
                smpl_thetas=np.array([rows[i][2] for i in order], F), smpl_betas=np.array([rows[i][3] for i in order], F),
                params_pred=np.array([rows[i][4] for i in order], F), pred_batch_ids=np.zeros(len(rows), np.int64))


def separated_video(seed, frames=180):
    """Four nearly static, well separated people and one-frame blips, all with high scores (so the second association
    never runs), laid out so that every lifecycle path of the tracker is taken (frame t is tracker frame t + 1):
      * person 1 is absent for 10 frames and is re-found from the lost list;
      * person 2 is absent for 61 frames: removed by age (more than 60 frames lost), still in the lost list on that
        frame, re-found from there on the next one; lost again later, it leaves the lost list at once (its id is in the
        removed list) and comes back under a new id;
      * person 3 is absent for 100 frames: removed by age, back under a new id;
      * blips at the centre start unconfirmed tracks that are removed on the next frame."""
    rs = np.random.RandomState(seed)
    anchors = [(0.42, -0.45, -0.45), (0.40, -0.45, 0.45), (0.44, 0.45, -0.45), (0.38, 0.45, 0.45)]
    absent = [[], [(30, 40)], [(50, 111), (150, 155)], [(60, 160)]]
    blips = {20, 45, 130}                            # frames with no lost track (a lost track would take a blip)
    th = [rs.normal(0, 0.3, 72) for _ in range(5)]
    be = [rs.normal(0, 0.4, 11) for _ in range(5)]
    pp = [rs.normal(0, 1, 146) for _ in range(5)]
    seq = []
    for t in range(frames):
        rows = []
        for p, a in enumerate(anchors):
            cam = np.array(a) + np.r_[rs.normal(0, 0.002), rs.normal(0, 0.002, 2)]
            th[p] += rs.normal(0, 0.02, 72)
            be[p] += rs.normal(0, 0.01, 11)
            if any(g0 <= t < g1 for g0, g1 in absent[p]):
                continue
            rows.append((cam, rs.uniform(0.3, 0.9), th[p].copy(), be[p].copy(), pp[p] + rs.normal(0, 0.01, 146)))
        if t in blips:
            rows.append((np.array([0.3, 0.0, 0.0]), 0.5, th[4].copy(), be[4].copy(), pp[4].copy()))
        seq.append(_frame_dict(rows, rs))
    return seq


def make_video(kind, seed, frames, people=(6, 12), empty_every=0):
    """kind 0: synthetic_video, kind 1: separated_video."""
    return synthetic_video(seed, frames, people, empty_every=empty_every) if kind == 0 else separated_video(seed, frames)


# ----------------------------------------------------------------------------------------------------------------
# Edge sequences: every decision of the tracker placed on, or one fp32 step from, its threshold.  Detections are given
# as tracking points; the inputs are chosen so that bev/main.py:269-272 gives each point back exactly in fp32.
# A fresh track has zero velocity, so its predicted mean is its fp32 point and a displacement of 300 along x is a cost
# of exactly 300.  Placements that depend on the Kalman filter are measured from this module's fp64 8x8 filter.
SPACING = 3000.0             # between anchors: farther than any limit, so only the intended pairs can ever match
HIGH, LOWS, NONE = F(0.5), F(0.08), F(0.03)      # a high score, a low one (runs the second matching), one that is neither


def up(x, k=1):
    for _ in range(k):
        x = np.nextafter(F(x), F(np.inf))
    return F(x)


def down(x, k=1):
    for _ in range(k):
        x = np.nextafter(F(x), F(-np.inf))
    return F(x)


def zfit(z):
    """The fp32 depth point cam_trans2 * 30 nearest z that an fp32 cam_trans2 reaches."""
    return F(F(F(z) / F(30)) * F(30))


def anchor(i, z=300.0, h=32.0):
    return np.array([1000 + SPACING * (i % 8), 1000 + SPACING * (i // 8), zfit(z), h], F)


def edge_point(center, lam, inside, dim=4, axis=0, sign=1):
    """The fp32 point on the line from ``center`` along ``axis`` nearest the threshold: its other coordinates are
    ``center``'s rounded to reachable fp32, and on the axis it is the farthest value whose fp64 distance (first ``dim``
    coordinates) is below lam (inside), or the nearest one above lam (outside).  Returns (point, distance)."""
    center = np.asarray(center, np.float64)
    p = center.astype(F)
    p[2] = zfit(center[2])
    dist = lambda q: float(np.linalg.norm(q[:dim].astype(np.float64) - center[:dim]))
    out_, in_ = (up, down) if sign > 0 else (down, up)
    p[axis] = F(center[axis] + sign * lam)
    while dist(p) >= lam:
        p[axis] = in_(p[axis])
    while True:
        q = p.copy()
        q[axis] = out_(q[axis])
        if dist(q) >= lam:
            break
        p = q
    if not inside:
        p = q
        while dist(p) <= lam:
            p[axis] = out_(p[axis])
    return p, dist(p)


def predicted(t):
    """The mean a listed track is matched with on the next stepped frame (unconfirmed tracks are not predicted)."""
    if not t.activated:
        return t.mean.copy()
    m = t.mean.copy()
    if t.state != TRACKED:
        m[7] = 0
    return _Fm @ m


class EdgeVideo:
    """Frames built one at a time while this module's tracker follows them, so that later placements can be measured
    from the filter.  ``ties``: frames holding an assignment tie that lapjv may break either way (a cost exactly at a
    limit, or two optimal matchings); ``broken``: the first frame on which a 128-entry track table is full."""

    def __init__(self, seed, show_largest=False):
        self.rs = np.random.RandomState(seed)
        self.frames, self.ties, self.broken, self.show_largest = [], [], None, show_largest
        self.tracker = Tracker()

    def add(self, dets, tie=False):
        """dets: [(point, score)], one frame; [] = a frame with nobody (it does not step the tracker)."""
        if tie:
            self.ties.append(len(self.frames))
        if not dets:
            self.frames.append({})
            return
        pts, sc = np.array([p for p, _ in dets], F), np.array([s for _, s in dets], F)
        n = len(pts)
        assert n <= 64 and (pts[:, :2] >= 128).all()
        cam = np.stack([pts[:, 3] / F(64), pts[:, 1] / F(128) - F(1), pts[:, 0] / F(128) - F(1)], 1).astype(F)
        ct = cam_to_trans(cam)
        for i in range(n):                                      # an fp32 cam_trans2 with cam_trans2 * 30 == z
            c = F(pts[i, 2] / F(30))
            c = next(v for v in (c, up(c), down(c), up(c, 2), down(c, 2)) if F(v * F(30)) == pts[i, 2])
            ct[i, 2] = c
        rs = self.rs
        f = dict(cam=cam, cam_trans=ct, center_confs=sc, smpl_thetas=rs.normal(0, 0.3, (n, 72)).astype(F),
                 smpl_betas=rs.normal(0, 0.4, (n, 11)).astype(F), params_pred=rs.normal(0, 1, (n, 146)).astype(F),
                 pred_batch_ids=np.zeros(n, np.int64))
        assert np.array_equal(tracking_points(f["cam"], f["cam_trans"]), pts)
        self.frames.append(f)
        if not self.show_largest:
            self.tracker.update(pts, sc)

    def track(self, tid):
        return next(t for t in self.tracker.tracked + self.tracker.lost if t.id == tid)

    def pred(self, tid):
        return predicted(self.track(tid))

    def newest(self, k=1):
        """ids of the k tracks created last"""
        return list(range(self.tracker.count - k + 1, self.tracker.count + 1))


def _scores(v):
    """conf at 0.12f and 0.05f and one fp32 step either side; then, frame by frame, the frame's only sub-0.12 detection
    decides whether the second matching (BT:75-80) runs for a track whose detection is 450 away."""
    ss = [DET_THRESH, up(DET_THRESH), down(DET_THRESH), LOW_THRESH, up(LOW_THRESH), down(LOW_THRESH)]
    v.add([(anchor(i), s) for i, s in enumerate(ss)] + [(anchor(8 + k), HIGH) for k in range(len(ss))])
    targets = v.newest(len(ss))                               # the anchors 8.. (and up(0.12) at anchor 1, created first)
    for k, s in enumerate(ss):                                 # frame 2 + k: anchor 8 + k's track tests score s
        dets = [(anchor(8 + j), HIGH) for j in range(len(ss)) if j > k]
        dets.append((anchor(8 + k) + np.array([450, 0, 0, 0], F), HIGH))
        dets.append((anchor(20 + k), s))
        v.add(dets)
    return targets


def _match(v):
    """For each matching, a detection one fp32 step inside and one step outside its limit: 300 against tracked tracks,
    600 against a tracked track the first matching left (with a low-score detection in the frame), 900 against an
    unconfirmed track created on frame 3."""
    v.add([(anchor(i), HIGH) for i in range(4)])             # tracks at anchors 0-3, activated
    d = lambda i, lam, inside: edge_point(anchor(i).astype(np.float64), lam, inside)[0]
    v.add([(d(0, 300, True), HIGH), (d(1, 300, False), HIGH), (anchor(2), HIGH), (anchor(3), HIGH)])
    v.add([(d(2, 600, True), HIGH), (d(3, 600, False), HIGH), (anchor(10), LOWS), (anchor(4), HIGH), (anchor(5), HIGH)])
    v.add([(d(4, 900, True), HIGH), (d(5, 900, False), HIGH)])
    v.add([(anchor(i), HIGH) for i in range(4)])


def _tie_limit(v, lam):
    """A cost exactly at the limit (300 and 900 on one frame, 600 on its own since it needs a low-score detection):
    lapjv's extended problem ties there; the rule checked is the documented one, the pair is dropped."""
    v.add([(anchor(0), HIGH), (anchor(1), HIGH)])
    v.add([(anchor(0), HIGH), (anchor(1), HIGH), (anchor(2), HIGH)])       # anchor 2: unconfirmed, created on frame 2
    off = lambda i, lam: anchor(i) + np.array([lam, 0, 0, 0], F)
    if lam == 600:
        v.add([(anchor(0), HIGH), (off(1, 600), HIGH), (anchor(12), LOWS)], tie=True)
    else:
        v.add([(off(0, 300), HIGH), (anchor(1), HIGH), (off(2, 900), HIGH)], tie=True)


def _kalman(v):
    """Tracks with 1 to 80 updates along paths whose scale mean[3] grows (8 to 88) or shrinks (96 to 16), some lost for a
    few frames (velocity zeroed) before their last detection.  That one is one fp32 step inside or outside 300 from the
    fp64 filter's prediction.  Two tracks end lost, with a new detection 60 px (2-D) from the predicted mean, one step
    inside or outside, 450 deeper: the new track is or is not a duplicate, which shows on the next frame (confirmed, with a
    row, or not).  Two end on two detections one fp32 step apart along x: the row takes the nearer (second) one."""
    rs = v.rs
    plans = []
    for k, (n, gap) in enumerate([(1, 0), (2, 0), (5, 3), (10, 0), (20, 6), (40, 2), (60, 0), (80, 4)]):
        for end in ("in", "out"):
            plans.append(dict(n=n, gap=gap, end=end, grow=k % 2 == 0))
    plans += [dict(n=12, gap=3, end="dup_in", grow=True), dict(n=12, gap=3, end="dup_out", grow=False),
              dict(n=9, gap=0, end="near_first", grow=True), dict(n=15, gap=0, end="near_second", grow=False)]
    for a, p in enumerate(plans):
        p["a"], p["e"] = a, p["n"] + p["gap"]
    ids, dup = {}, {}
    for t in range(max(p["e"] for p in plans) + 2):
        dets = []
        for p in plans:
            a = p["a"]
            if t < p["n"]:                                     # the path, detected with noise
                h = 8.0 + t if p["grow"] else 96.0 - t
                pt = anchor(a, z=300.0 + 0.5 * t, h=h) + np.array([3.0 * t, -2.0 * t, 0, 0]) + rs.normal(0, [1.5, 1.5, 0, 0.2])
                pt[2] = zfit(pt[2])
                dets.append((pt.astype(F), HIGH))
            elif t == p["e"] and p["end"] in ("in", "out"):
                dets.append((edge_point(v.pred(ids[a])[:4], MATCH, p["end"] == "in", sign=1 if a % 4 < 2 else -1)[0], HIGH))
            elif t == p["e"] and p["end"].startswith("dup"):
                q, _ = edge_point(v.pred(ids[a])[:4], DUP, p["end"] == "dup_in", dim=2)
                q[2] = zfit(q[2] + 450)
                dup[a] = q
                dets.append((q, HIGH))
            elif t == p["e"] + 1 and p["end"].startswith("dup"):
                dets.append((dup[a], HIGH))
            elif t == p["e"] and p["end"].startswith("near"):
                d = v.pred(ids[a])[:4].astype(F)
                d[2], d[0] = zfit(d[2]), F(d[0] + 20)
                dets += [(d, HIGH), (np.r_[down(d[0]) if p["end"] == "near_second" else up(d[0]), d[1:]].astype(F), HIGH)]
        v.add(dets)
        if t == 0:
            ids = dict(zip(range(len(plans)), v.newest(len(plans))))


def _dup(v):
    """Duplicate removal (BT:187-201) between fresh tracks, whose means are their fp32 points: a lost track of age 0 and
    a new one 450 deeper at 2-D distance exactly 60, one fp32 step inside, one step outside; the equal ages remove the
    tracked one (it never gets a row); a new track next to an older lost one is removed, one next to a younger lost one
    removes that instead."""
    off = lambda i, dx: anchor(i) + np.array([dx, 0, 450, 0], F)
    v.add([(anchor(i), HIGH) for i in range(5)])             # frame 1: five tracks, activated, age 0
    v.add([(anchor(5), HIGH), (anchor(4), HIGH)])            # they are lost, anchor 4 ages to 1
    v.add([(off(0, 60.0), HIGH), (off(1, down(F(1060)) - 1000), HIGH), (off(2, up(F(1060)) - 1000), HIGH), (anchor(5), HIGH)])
    v.add([(off(0, 60.0), HIGH), (off(1, down(F(1060)) - 1000), HIGH), (off(2, up(F(1060)) - 1000), HIGH), (anchor(5), HIGH),
           (off(3, 30.0), HIGH)])                             # exactly 60: kept, confirmed; anchor 3: equal ages
    v.add([(off(i, d), HIGH) for i, d in ((0, 60.0), (2, up(F(1060)) - 1000), (3, 30.0))] + [(anchor(5), HIGH)])


def _lifecycle(v):
    """Removal after more than 60 lost frames (BT:122-125), counted in stepped frames: frames with nobody in between do
    not step the tracker (bev/main.py:159-163).  Tracks lost on frame 2 come back on stepped frame 61 (lost exactly 60
    frames), 62 (re-found just before removal), 63 (removed on 62, still listed, re-found from there; lost again on 64,
    it leaves the lists at once and its return on 65 is a new track) and 64 (gone: a new track)."""
    keep = lambda: (anchor(0), HIGH)
    v.add([keep()] + [(anchor(i), HIGH) for i in range(1, 5)])
    back = {61: [1], 62: [2], 63: [3], 64: [4], 65: [3]}
    fid, t = 1, 0
    while fid < 66:
        t += 1
        if t % 9 == 4:
            v.add([])                                        # nobody: not a tracker step
            continue
        fid += 1
        v.add([keep()] + [(anchor(i), HIGH) for i in back.get(fid, [])])


def _ties(v):
    """Nearest-detection ties (BT:149-159: np.argmin, the first on ties): two tracks started on one point share its first
    detection; a matched track with an identical detection listed before its own takes that one."""
    v.add([(anchor(0), HIGH), (anchor(0), HIGH), (anchor(1), HIGH), (anchor(2), HIGH)])
    d = anchor(1) + np.array([5, 5, 0, 1], F)
    v.add([(anchor(2), HIGH), (d, HIGH), (d, HIGH), (anchor(0), HIGH)])
    v.add([(anchor(9), HIGH), (anchor(2), HIGH), (anchor(0), HIGH), (anchor(0), HIGH), (anchor(2), HIGH), (d, HIGH)])


def _largest(v):
    """--show_largest: torch.argmax(cam[:, 0]), the first on ties, and the larger of two values one fp32 step apart."""
    h = lambda c0: np.r_[anchor(0)[:3], F(c0) * F(64)].astype(F)
    for cams in ([0.5, 0.5, 0.4], [0.3, 0.5, 0.5], [0.4, float(up(F(0.4))), 0.4], [float(up(F(0.4))), 0.4, 0.4],
                 [0.2, 0.2, 0.2, 0.2], [0.25]):
        v.add([(np.r_[anchor(k)[:3], F(c) * F(64)].astype(F), HIGH) for k, c in enumerate(cams)])


def _assign128(v):
    """128 live tracks and a 64-detection frame: the first matching is 128 x 64.  16 clusters of 4 + 4 tracks (4 started
    on frame 1, 4 on frame 2, 320 deeper so that nothing matches across and 90 px aside so that neither is a duplicate of
the other) and, on the last frame, 4 detections half way,
    every cost in a cluster a random real below 300.  Frames whose only detection scores 0.03 step the tracker and leave
    every track lost, so the filter gain is near 1 and each row's nearest detection is its matched one.  The optimum is
    unique by a margin the generator checks."""
    rs = v.rs
    while True:
        a = [[np.r_[rs.uniform(-75, -45), rs.uniform(-40, 40), 0, rs.uniform(-6, 6)] for _ in range(4)] for _ in range(16)]
        b = [[np.r_[rs.uniform(45, 75), rs.uniform(-40, 40), 320, rs.uniform(-6, 6)] for _ in range(4)] for _ in range(16)]
        d = []
        while len(d) < 16:                                  # detections of a cluster at least 40 apart
            c4 = [np.r_[rs.uniform(-40, 40, 2), 160 + rs.uniform(-20, 20), rs.uniform(-6, 6)] for _ in range(4)]
            if min(np.linalg.norm(x - y) for x, y in itertools.combinations(c4, 2)) > 41:
                d.append(c4)
        pt = lambda k, o: (anchor(k, z=300.0 + o[2], h=32.0 + o[3]) + np.r_[o[:2], 0, 0]).astype(F)
        A = np.array([pt(k, o) for k in range(16) for o in a[k]])
        B = np.array([pt(k, o) for k in range(16) for o in b[k]])
        D = np.array([pt(k, o) for k in range(16) for o in d[k]])
        A[:, 2], B[:, 2], D[:, 2] = (np.array([zfit(z) for z in X[:, 2]]) for X in (A, B, D))
        c = _dist(list(np.r_[A, B].astype(np.float64)), list(D.astype(np.float64)))
        same = np.repeat(np.arange(16), 4)
        within = np.r_[same, same][:, None] == same[None]
        dd = _dist(list(D.astype(np.float64)), list(D.astype(np.float64))) + np.eye(64) * 1e9
        if c[within].max() < MATCH - 5 and dd.min() > 40 and assignment_margin(c, MATCH) > 1e-3:
            break
    v.add([(p, HIGH) for p in A])
    v.add([(p, HIGH) for p in B])
    v.add([(p, HIGH) for p in B])
    for _ in range(5):
        v.add([(anchor(63), NONE)])
    v.add([(p, HIGH) for p in D])


def assignment_margin(cost, lam):
    """How much worse the best extended assignment is that avoids one pair of the optimum (the gap to the runner-up)."""
    best, _, _ = lap_extended(cost, lam)
    val = lambda m, n_a, n_b: sum(cost[i, j] for i, j in m) + (n_a + n_b) * lam / 2
    v0 = val(best, cost.shape[0] - len(best), cost.shape[1] - len(best))
    gap = np.inf
    for i, j in best:
        c = cost.copy()
        c[i, j] = 1e9
        m, ua, ub = lap_extended(c, lam)
        gap = min(gap, val(m, len(ua), len(ub)) - v0)
    return gap


def _assign_tie(v):
    """Two optimal matchings of equal cost: tracks at (-60, 0) and (60, 0) from a centre, detections at (0, 80) and
    (0, -80), all four costs exactly 100."""
    c = anchor(0)
    v.add([(c + np.array([-60, 0, 0, 0], F), HIGH), (c + np.array([60, 0, 0, 0], F), HIGH), (anchor(1), HIGH)])
    v.add([(c + np.array([0, 80, 0, 0], F), HIGH), (c + np.array([0, -80, 0, 0], F), HIGH), (anchor(1), HIGH)], tie=True)


def _rows126(v):
    """The most rows one frame can emit: 63 high-score detections and one low-score one, 63 lost tracks re-found on
    them by the first matching and 63 tracked ones 400 away matched to the same detections by the second (every row
    shares its detection with another).  A frame cannot emit more: M1 + M3 <= nh and M2 <= nh, with nh <= 63 whenever the
    second matching runs.  Then two new tracks fill the table to 128, and a third one on the next frame finds no free
    entry."""
    P = [anchor(i) for i in range(63)]
    Q = [p + np.array([400, 0, 0, 0], F) for p in P]
    v.add([(p, HIGH) for p in P])                            # 63 tracks, activated
    v.add([(q, HIGH) for q in Q[:32]])                       # all lost; 32 new
    v.add([(q, HIGH) for q in Q])                            # 32 confirmed, 31 new
    v.add([(q, HIGH) for q in Q])                            # 31 confirmed
    v.add([(p, HIGH) for p in P] + [(anchor(63), LOWS)])     # 126 rows
    r = lambda i: anchor(63) - np.array([400 * (i + 1), 0, 0, 0], F)
    v.add([(r(0), HIGH), (r(1), HIGH)])                     # all 126 lost (neither list is tracked: no duplicates), 128
    v.broken = len(v.frames)
    v.add([(r(0), HIGH), (r(1), HIGH), (r(2), HIGH)])        # a 129th track


# kind -> (builder, show_largest)
EDGE_KINDS = {"scores": (_scores, False), "match": (_match, False), "tie_limit": (lambda v: _tie_limit(v, 300), False),
              "tie_limit600": (lambda v: _tie_limit(v, 600), False), "kalman": (_kalman, False), "dup": (_dup, False),
              "lifecycle": (_lifecycle, False), "ties": (_ties, False), "largest": (_largest, True),
              "assign128": (_assign128, False), "assign_tie": (_assign_tie, False), "rows126": (_rows126, False)}


def edge_video(kind):
    """-> EdgeVideo of the named edge sequence (``.frames`` in make_video's format, ``.ties``, ``.broken``)."""
    build, largest = EDGE_KINDS[kind]
    v = EdgeVideo(sorted(EDGE_KINDS).index(kind), show_largest=largest)
    build(v)
    return v
