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
def lap_extended(cost, lam):
    """lap.lapjv(cost, extend_cost=True, cost_limit=lam) as linear_assignment uses it: the (n+m)^2 problem with the
    cost in the top-left block, lam/2 in both off-diagonal blocks and 0 in the dummy block.  Returns (matches [(i, j)],
    unmatched rows ascending, unmatched columns ascending)."""
    n, m = cost.shape
    if n == 0 or m == 0:
        return [], list(range(n)), list(range(m))
    ext = np.full((n + m, n + m), lam / 2.0)
    ext[:n, :m] = cost
    ext[n:, m:] = 0.0
    r, c = linear_sum_assignment(ext)
    x = np.full(n, -1)
    y = np.full(m, -1)
    for i, j in zip(r, c):
        if i < n and j < m:
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
    z = np.asarray(z, np.float64)
    h = z[3]
    std = np.r_[[2 * STD_POS * h] * 4, [10 * STD_VEL * h] * 4]
    return np.r_[z, np.zeros(4)], np.diag(std * std)


def kf_predict(mean, P):
    h = mean[3]
    q = np.r_[[STD_POS * h] * 4, [STD_VEL * h] * 4]
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


def _joint(a, b):
    ids = {t.id for t in a}
    return a + [t for t in b if t.id not in ids]


def _sub(a, b):
    ids = {t.id for t in b}
    return [t for t in a if t.id not in ids]


class Tracker:
    """Tracker(det_thresh=0.12, low_conf_det_thresh=0.05, track_buffer=60, match_thresh=300, frame_rate=30), BT:6-147.
    Ids count from 1 per instance.  ``margins`` collects (kind, distance to the threshold) of every decision."""

    def __init__(self):
        self.tracked, self.lost = [], []
        self.frame_id, self.count = 0, 0
        self.margins = []
        self.events = collections.Counter()          # refind, refind_removed, aged, unconfirmed_removed, lost_in_removed

    def _assign(self, tracks, dets, lam):
        c = _dist([t.point for t in tracks], [d.point for d in dets])
        if c.size:
            self.margins.append(("match", float(np.abs(c - lam).min()) / lam))
        return lap_extended(c, lam)

    def update(self, points, scores):
        """points fp32 [N,4], scores fp32 [N] -> (track ids, detection index per row)."""
        points, scores = np.asarray(points, F), np.asarray(scores, F)
        self.frame_id += 1
        fid = self.frame_id
        if len(scores):
            self.margins.append(("score", float(min(np.abs(scores - DET_THRESH).min(), np.abs(scores - LOW_THRESH).min()))))
        high = scores > DET_THRESH
        low = (scores > LOW_THRESH) & (scores < DET_THRESH)
        dets = [Track(p, s) for p, s in zip(points[high], scores[high])]
        activated, refind, lost_new, removed_new = [], [], [], []
        unconfirmed = [t for t in self.tracked if not t.activated]
        pool = _joint([t for t in self.tracked if t.activated], self.lost)
        for t in pool:                                                         # STrack.multi_predict
            m = t.mean.copy()
            if t.state != TRACKED:
                m[7] = 0
            t.mean, t.P = kf_predict(m, t.P)

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
            if fid - t.frame_id > MAX_LOST:
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
        for p, q in zip(*np.where(pd < DUP)):
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
            inds.append(int(np.argmin(d)))
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

    def __init__(self, show_largest=False, smooth_coeff=3.0):
        self.show_largest, self.smooth_coeff = show_largest, smooth_coeff
        self.tracker = None if show_largest else Tracker()
        self.filters = {}

    def __call__(self, out, signal_ID=0):
        """out: numpy dict of the result_keys for one frame with at least one detection.  Returns the smoothed dict
        (cam_trans recomputed from the smoothed cam, bev/main.py:169), or None."""
        out = {k: np.array(v) for k, v in out.items()}
        if self.show_largest:
            f = self.filters.setdefault(signal_ID, T.make_filters(self.smooth_coeff))
            k = int(np.argmax(out["cam"][:, 0]))
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
