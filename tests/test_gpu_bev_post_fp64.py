"""BEV's stages after SMPL, each run through the C ABI on crafted device inputs and compared with a plain float64
restatement of the reference's formulas written here (bev/post_parser.py:68-222, bev/main.py:179-256):
  b200romp_bev_post(_frames)   projection (pj2d_org against float64, per-element bounds), then per frame the scale-based
                               suppression and remove_outlier: the kept rows, frames of 0 .. 64 rows (CAP 64) and of 128
                               rows (CAP 128, video mode); _post_frames bit-equal to _post per frame
  b200romp_bev_crop_post       the 22 crops of a 1080 x 3840 image in two chunks: boundary drop at each finite limit of
                               the crop table and one float either side (crops 0, 1, the middle and the last),
                               conf-based suppression, remove_outlier(scale_thresh=1), cam_full bit for bit, survivors
                               appended bit-equal to their rows, and an acc_capacity that cuts the second chunk
  b200romp_bev_long_merge      cam_trans, pj2d_org, the kept rows at 0 .. 1407 accumulated persons, and the per-survivor
                               mean distances read from the workspace against float64
  b200romp_gather_rows         row copies of 4 .. 82,680 bytes
Joints, cam, cam_trans and conf are crafted directly; SMIL is skipped (verts_smil = joints_smil = NULL).

Decisions.  Each pair test dn < thr and each outlier test rel > relative_scale_thresh gets from the float64 restatement
its margin and a bound on what a correct fp32 evaluation of the reference's formula can be off by (71 norms and their
mean for dn; the sorted-row mean, the sum of the means and the cancellation in tot - mean_i for rel).  Where the margin
exceeds the bound the kernel's decision must be float64's; the others are enumerated, and the kernel's kept rows must
equal float64's pipeline under one resolution of them (suppression feeds remove_outlier, so every branch is carried
through).  Ties are pinned: equal scale or conf removes the later person, a pair test is <, remove_outlier runs at n >= 3.
One frame puts a decision inside its bound on purpose: its persons are spaced so that none is suppressed, and one of
them is moved along its viewing ray until its float64 rel lands on float32(relative_scale_thresh); the test asserts it
stays inside the bound.
The threshold itself is pinned exactly: with one joint apart and both persons on one image row, the kernel's normalised
distance is |dx| / 71 / max_scale with two roundings only, whatever the summation order; the scale is chosen so that it
lands on float32(thresh * max(h, w, 3) / 640) and on the floats either side.

Values are checked per element, |err| <= g * 2^-24 * cond, cond the restatement on absolute values; each check prints
its worst err / bound.  Output buffers are pre-filled with a sentinel, rows past the count must keep it bit for bit.
Negative controls mutate the restatement and must be rejected.  The tests without the gpu marker run fp32 emulations of
the kernels through the same checks: the reference's sorted-row mean is accepted, the (sum - min - max) mean the kernels
used before is rejected on a far outlier, and each mutant of the decision rules is rejected.

Worst err / bound on an H100 80 GB HBM3 at 700 W: pj2d_org 0.30 (CAP 64, CAP 128, crops), long-merge cam_trans 0.37
and pj2d_org 0.30, row means of remove_outlier 0.19 at 3 survivors and 0.002 at 1271.  With the (sum - min - max) row
mean the kernels used before, the long merge's row means fail by 10x to 34x at 3 to 16 survivors (the person at depth
4e4); every decision of the file, the tuned inlier's included, still passes: that formula's error there is far inside
the bound of a correct fp32 evaluation (0.001 of it for the tuned inlier), so only the row-mean check tells the two
apart.  The fp32 emulation gives 30x and 3300x on the far-outlier rows at depth 1e3 and 4e4.  The GPU tests of this file
take about 10 s and peak at 228 MiB of device memory."""
import ctypes as C
import itertools

import numpy as np
import pytest
import torch

from romp_b200 import _lib
from romp_b200.bev import long_image_crop_table, long_image_plan

gpu = pytest.mark.gpu
P = lambda t: C.c_void_p(t.data_ptr())
U = 2.0 ** -24
TINY = 1e-30
SENT = -7
F32, F64 = np.float32, np.float64
NJ = 71
C443, E6, E3, TAN = F32(443.4), F32(1e-6), F32(1e-3), F32(np.tan(np.radians(30.0)))
REL_T = 1.6                 # relative_scale_thresh of BEV's default settings
G_DN = NJ + 8               # 71-term mean of norms (3 roundings each), two divisions
G_PROJ = 2.0                # first-order projection bound, doubled
G_TRANS = 2.0
SIZES = [(1, 1), (2, 2), (2, 301), (37, 53), (1080, 1920), (1920, 1080)]


def stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def report(name, err, bound):
    """err <= bound everywhere (a NaN fails); prints and returns the worst ratio."""
    err, bound = np.asarray(err, F64), np.asarray(bound, F64) + TINY
    ratio = float(np.max(err / bound)) if err.size else 0.0
    print(f"{name}: max|err| {float(np.max(err)) if err.size else 0.0:.3e}  worst err/bound {ratio:.3f}")
    return ratio if np.all(err <= bound) else float("inf")


def accepted(name, err, bound):
    r = report(name, err, bound)
    assert r <= 1.0, f"{name}: outside the bound or not finite"
    return r


def rejected(name, err, bound):
    r = report("  control " + name, err, bound)
    assert r > 1.0, f"negative control {name} was not rejected"


@pytest.fixture(scope="module", autouse=True)
def peak_memory():
    yield
    if torch.cuda.is_available():
        print(f"\npeak device memory of this file: {torch.cuda.max_memory_allocated() / 2 ** 20:.0f} MiB")


# ============================================================================================ float64 restatement
def thr_px(nms, max_side, mutate=None):
    """the fp32 number torch compares with: float32(thresh * max(img_shape) / 640), img_shape = (h, w, 3)."""
    max_side = float(max_side)                      # a numpy float32 side would make the product float32
    if mutate == "no3":
        return F64(F32(nms * max_side / 640))
    if mutate == "float_thr":
        return F64(F32(F32(F32(nms) * F32(max_side)) / F32(640)))
    return F64(F32(nms * max(max_side, 3) / 640))


def project64(joints, ct, size, left, top):
    """perspective_projection + convert_proejection_from_input_to_orgimg in float64 -> (pj [n,71,2], bound)."""
    j, t = joints.astype(F64), ct.astype(F64)[:, None, :]
    p = j + t
    iz = p[..., 2] + F64(E6)
    a_iz = np.abs(j[..., 2]) + np.abs(t[..., 2]) + F64(E6)
    out, bnd = [], []
    for c, off in ((0, left), (1, top)):
        q = p[..., c] / iz
        e_q = U * ((np.abs(j[..., c]) + np.abs(t[..., c])) / np.abs(iz) + np.abs(q) * a_iz / np.abs(iz) + np.abs(q))
        uu = q * F64(C443) / 256.0
        e_u = e_q * F64(C443) / 256.0 + U * np.abs(uu)
        w = (uu + 1.0) * F64(size) / 2.0
        e_w = (e_u + U * (np.abs(uu) + 1.0)) * F64(size) / 2.0 + U * np.abs(w)
        pj = w - F64(off)
        out.append(pj)
        bnd.append(G_PROJ * (e_w + U * (np.abs(w) + abs(F64(off)))))
    return np.stack(out, -1), np.stack(bnd, -1)


def cam_trans64(cam):
    """denormalize_cam_params_to_trans with torch's fp32 constants, float64 -> (trans [n,3], bound)."""
    c = cam.astype(F64)
    den = c[:, 0] * F64(TAN) + F64(E3)
    depth = 1.0 / den
    e_depth = np.abs(depth) * U * ((np.abs(c[:, 0] * F64(TAN)) * 2 + F64(E3)) / np.abs(den) + 1.0)
    tx, ty = c[:, 2] * depth * F64(TAN), c[:, 1] * depth * F64(TAN)
    e = lambda v, cc: np.abs(cc * F64(TAN)) * e_depth + 2 * U * np.abs(v)
    tr = np.stack([tx, ty, depth], 1)
    return tr, G_TRANS * np.stack([e(tx, c[:, 2]), e(ty, c[:, 1]), e_depth], 1)


def dn_matrix(pj):
    """normalised-distance numerators: mean over the 71 joints of the 2-D norm, float64, [n,n]."""
    pj = pj.astype(F64)
    n = len(pj)
    out = np.zeros((n, n))
    for r0 in range(0, n, 32):
        d = pj[r0:r0 + 32, None] - pj[None]
        out[r0:r0 + 32] = np.sqrt((d * d).sum(-1)).mean(-1)
    return out


def pair_decisions(pj, cam0, conf, conf_based, thr, drop, mutate=None, dist=None):
    """-> (removed for sure, ambiguous [(i, j, victim)]) of the suppression over the non-dropped persons."""
    n = len(cam0)
    dist = dn_matrix(pj) if dist is None else dist
    s = cam0.astype(F64) * 2
    ii, jj = np.triu_indices(n, 1)
    if mutate != "keep_dropped":
        m = ~(drop[ii] | drop[jj])
        ii, jj = ii[m], jj[m]
    with np.errstate(divide="ignore", invalid="ignore"):
        dn = dist[ii, jj] / np.maximum(s[ii], s[jj])
    bound = G_DN * U * np.abs(dn)
    below = dn <= thr if mutate == "le" else dn < thr
    amb = np.abs(dn - thr) <= bound
    use_conf = conf_based != (mutate == "swap_rules")
    key = conf.astype(F64) if use_conf else s
    first = key[ii] < key[jj]
    if mutate == "tie_reversed":
        first = key[ii] <= key[jj]
    victim = np.where(first, ii, jj)
    sure = set(victim[below & ~amb].tolist())
    return sure, [(int(a), int(b), int(v)) for a, b, v in zip(ii[amb], jj[amb], victim[amb])]


def outlier_stats(ct):
    """remove_outlier's float64 row means, rel, and the fp32 bounds of both (the reference's formula)."""
    t = ct.astype(F64)
    n = len(t)
    d = np.sqrt(((t[:, None] - t[None]) ** 2).sum(-1))
    mean = np.sort(d, 1)[:, 1:-1].mean(1)
    e_mean = (n + 4) * U * mean
    tot = mean.sum()
    e_tot = (n - 1) * U * tot + e_mean.sum()
    num = tot - mean
    den = num / (n - 1)
    e_den = (U * np.abs(num) + e_tot + e_mean) / (n - 1) + U * np.abs(den)
    with np.errstate(divide="ignore", invalid="ignore"):
        rel = mean / den
        e_rel = np.abs(rel) * (np.where(mean > 0, e_mean / mean, 0) + e_den / np.abs(den) + 2 * U) * 1.01
    return mean, e_mean, rel, e_rel


def outlier_sets(ct, cam0, rel_t, scale_t, mutate=None):
    """every kept-index list remove_outlier can give under the fp32 bounds of its rel tests."""
    n = len(ct)
    if n < 3:
        return [list(range(n))]
    _, _, rel, e_rel = outlier_stats(ct)
    small = cam0 < F32(scale_t)
    thr = F64(F32(rel_t))
    out = small & (rel > thr)
    amb = small & (np.abs(rel - thr) <= e_rel)
    idx = np.flatnonzero(amb)
    assert len(idx) <= 8, f"{len(idx)} ambiguous outlier tests"
    res = []
    for bits in itertools.product([0, 1], repeat=len(idx)):
        o = out.copy()
        o[idx] = np.array(bits, bool)
        res.append([i for i in range(n) if not o[i]])
    return res


def frame_sets(pj, cam, ct, conf, conf_based, thr, rel_t, scale_t, drop=None, mutate=None, dist=None):
    """every kept-index set of one frame's two filters under one resolution of its ambiguous decisions."""
    n = len(cam)
    drop = np.zeros(n, bool) if drop is None else drop
    if n == 1 and mutate != "keep_dropped":
        return {tuple(i for i in range(n) if not drop[i])}
    sure, amb = pair_decisions(pj, cam[:, 0], conf, conf_based, thr, drop, mutate, dist) if n > 1 else (set(), [])
    assert len(amb) <= 8, f"{len(amb)} ambiguous pair tests"
    sets = set()
    for bits in itertools.product([0, 1], repeat=len(amb)):
        removed = sure | {v for (_, _, v), b in zip(amb, bits) if b}
        k1 = [i for i in range(n) if i not in removed and (mutate == "keep_dropped" or not drop[i])]
        for k2 in outlier_sets(ct[k1], cam[k1, 0], rel_t, 0.25 if mutate == "scale_quarter" else scale_t, mutate):
            sets.add(tuple(i for i in (k1[j] for j in k2) if not drop[i]))
    return sets


# ================================================================================= fp32 emulations of the kernels
def project32(joints, ct, size, left, top):
    """bev_project_kernel's fp32 op order (bit-exact with the kernel)."""
    px = joints[..., 0] + ct[:, None, 0]
    py = joints[..., 1] + ct[:, None, 1]
    iz = (joints[..., 2] + ct[:, None, 2]) + E6
    u = (px / iz) * C443 / F32(256)
    v = (py / iz) * C443 / F32(256)
    return np.stack([(u + F32(1)) * F32(size) / F32(2) - F32(left), (v + F32(1)) * F32(size) / F32(2) - F32(top)], -1)


def cam_trans32(cam):
    depth = F32(1) / (cam[:, 0] * TAN + E3)
    return np.stack([(cam[:, 2] * depth) * TAN, (cam[:, 1] * depth) * TAN, depth], 1).astype(F32)


def row_means32(ct, formula):
    """fp32 row means of remove_outlier: 'sort' the reference's sorted row, 'maxskip' the kernels' row without its first
    maximum, 'summinmax' (sum - min - max) as the kernels computed it before."""
    n = len(ct)
    out = np.zeros(n, F32)
    for i in range(n):
        d = ct[i] - ct
        r = np.sqrt(d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1] + d[:, 2] * d[:, 2]).astype(F32)
        if formula == "sort":
            vals = np.sort(r)[1:-1]
        elif formula == "maxskip":
            vals = np.delete(r, int(np.argmax(r)))
        else:
            vals = None
        s = F32(0)
        for x in (r if vals is None else vals):
            s = F32(s + x)
        if vals is None:
            s = F32(F32(s - r.min()) - r.max())
        out[i] = s / F32(n - 2)
    return out


def frame_emulate32(pj, cam, ct, conf, conf_based, thr, rel_t, scale_t, drop=None, formula="maxskip"):
    """postfilter_frame in fp32 -> (kept indices, row means of the outlier step or None)."""
    n = len(cam)
    drop = np.zeros(n, bool) if drop is None else drop
    removed = drop.copy()
    thr32 = F32(thr)
    for i in range(n):
        for j in range(i + 1, n):
            if drop[i] or drop[j]:
                continue
            s = F32(0)
            for k in range(NJ):
                dx, dy = F32(pj[i, k, 0] - pj[j, k, 0]), F32(pj[i, k, 1] - pj[j, k, 1])
                s = F32(s + np.sqrt(F32(dx * dx + dy * dy)))
            si, sj = F32(cam[i, 0] * 2), F32(cam[j, 0] * 2)
            with np.errstate(divide="ignore", invalid="ignore"):
                below = F32(F32(s / F32(NJ)) / max(si, sj)) < thr32
            if below:
                first = conf[i] < conf[j] if conf_based else si < sj
                removed[i if first else j] = True
    k = [i for i in range(n) if not removed[i]]
    if len(k) < 3:
        return k, None
    m = row_means32(ct[k], formula)
    tot = F32(0)
    for x in m:
        tot = F32(tot + x)
    rel = m / ((tot - m) / F32(len(k) - 1))
    out = (rel > F32(rel_t)) & (cam[k, 0] < F32(scale_t))
    return [i for i, o in zip(k, out) if not o], m


# ============================================================================================= crafted frames
def body(rs, n, spread=0.3):
    base = rs.normal(0, spread, (1, NJ, 3)).astype(F32)
    return (base + rs.normal(0, 0.02, (n, NJ, 3))).astype(F32)


def crowd(rs, n, dup=0.15):
    """n persons in front of the camera, some near-duplicates (suppressed), cam[:,0] on both sides of 0.25."""
    joints = body(rs, n)
    ct = np.stack([rs.uniform(-2, 2, n), rs.uniform(-1, 1, n), rs.uniform(4, 14, n)], 1).astype(F32)
    cam = np.stack([rs.uniform(0.1, 0.6, n), rs.uniform(-1, 1, n), rs.uniform(-1, 1, n)], 1).astype(F32)
    for i in np.flatnonzero(rs.uniform(size=n) < dup)[1:]:
        ct[i] = ct[i - 1] + rs.normal(0, 0.01, 3).astype(F32)
    return joints, cam, ct


def far_outlier(rs, depth=4e4, n_in=4):
    """n_in persons within about 0.5 of each other and one more at the given depth (scale below 0.25)."""
    joints = body(rs, n_in + 1)
    ct = np.concatenate([rs.uniform(-0.25, 0.25, (n_in, 3)) + [0, 0, 6], [[0.3, 0.1, depth]]]).astype(F32)
    cam = np.stack([np.r_[rs.uniform(0.3, 0.5, n_in), 0.1], rs.uniform(-1, 1, n_in + 1), rs.uniform(-1, 1, n_in + 1)], 1)
    return joints, cam.astype(F32), ct


def tuned_inlier(rs, rel_t=REL_T):
    """40 persons of a 1080 x 1920 frame: 38 on a grid spaced so that no pair is suppressed (every person reaches
    remove_outlier), a moderate outlier at depth 60, and person 1 moved along its viewing ray (its pixels stay put, clear
    of the others) until its float64 rel lands on float32(rel_t).  Both are small-scale, so both tests decide."""
    gx, gy = np.meshgrid(np.arange(-3.5, 4) * 0.5, np.arange(-2, 3) * 0.5)
    n = gx.size
    joints = body(rs, n, 0.15)
    ct = np.stack([gx.ravel(), gy.ravel(), np.full(n, 7.0)], 1).astype(F32)
    cam = np.stack([rs.uniform(0.3, 0.6, n), rs.uniform(-1, 1, n), rs.uniform(-1, 1, n)], 1).astype(F32)
    ct[0] = [30.0, 0.0, 60.0]
    cam[0, 0] = cam[1, 0] = 0.1
    ray = np.array([0.4, 0.4, 1.0])

    def ct_at(lam):
        c = ct.copy()
        c[1] = (lam * ray).astype(F32)
        return c
    lo, hi = 7.0, 300.0
    for _ in range(80):
        mid = 0.5 * (lo + hi)
        lo, hi = (mid, hi) if outlier_stats(ct_at(mid))[2][1] < F64(F32(rel_t)) else (lo, mid)
    return joints, cam, ct_at(hi)


TUNED = 8           # index of the tuned-inlier frame in post_frames


def tuned_margin(pj, cam, ct, thr, rel_t=REL_T):
    """the tuned frame: no pair test near or below its threshold, so all persons reach remove_outlier; returns
    |rel - thr| / bound of person 1 (float64 against the fp32 bound of the reference's formula)."""
    sure, amb = pair_decisions(pj, cam[:, 0], None, False, thr, np.zeros(len(cam), bool))
    assert not sure and not amb, "the tuned frame must reach remove_outlier whole"
    _, _, rel, e_rel = outlier_stats(ct)
    return abs(rel[1] - F64(F32(rel_t))) / e_rel[1]


def ties_and_scales(rs):
    """scales 0, negative and tied; two persons at one cam_trans (a distance row with two zeros)."""
    joints, cam, ct = crowd(rs, 7, dup=0.0)
    cam[:, 0] = [0.0, -0.1, 0.3, 0.3, 0.2, 0.2, 0.45]
    ct[3], joints[3] = ct[2], joints[2]            # equal scale, identical pixels: the later one goes
    ct[5] = ct[4]                                  # same cam_trans, different joints: two zeros in their rows
    joints[5] = joints[4] + F32(0.05)
    return joints, cam, ct


def placement_pool():
    """eight persons on one image row, all joints identical except joint 0 of persons 1.., further right by different
    amounts; two of them make a pair whose distance can be placed on a chosen float."""
    joints = np.zeros((8, NJ, 3), F32)
    joints[1:, 0, 0] = 0.3 + F32(0.037) * np.arange(1, 8, dtype=F32)
    ct = np.tile(np.array([[0.1, 0.2, 5.0]], F32), (8, 1))
    cam = np.tile(np.array([[0.1, 0.0, 0.0]], F32), (8, 1))
    return joints, cam, ct


def place_scale(pj, target):
    """max_scale m (= 2 cam[:,0] of both) so that the kernel's fp32 |dx| / 71 / m is exactly `target`, or None: the
    only other norms are 0, so the sum is |dx| in any order and the mean |dx| / 71 has one rounding."""
    assert pj[1, 0, 1] == pj[0, 0, 1] and np.array_equal(pj[0, 1:], pj[1, 1:])
    M = F32(abs(F32(pj[1, 0, 0] - pj[0, 0, 0])) / F32(NJ))
    up = down = F32(M / F32(target))
    for _ in range(64):
        for mc in (up, down):
            if F32(M / mc) == F32(target):
                return mc
        up, down = np.nextafter(up, F32(np.inf)), np.nextafter(down, F32(0))
    return None


def dn32_exact(pj, m):
    return F32(F32(abs(F32(pj[1, 0, 0] - pj[0, 0, 0])) / F32(NJ)) / F32(m))


def pad_row(h, w):
    s = max(h, w)
    return [(s - h) // 2, (s - h) // 2 + h, (s - w) // 2, (s - w) // 2 + w, h, w]


def frame(joints, cam, ct, hw):
    return dict(joints=joints, cam=cam, ct=ct, hw=hw)


def post_frames(seed, n_big=64):
    """batch of 32: frames of 0, 1, 2, 3 and n_big rows, far outliers, ties, a tuned inlier, depths near 0 and below."""
    rs = np.random.RandomState(seed)
    sz = lambda i: SIZES[i % len(SIZES)]
    fr = [frame(*crowd(rs, n), sz(n)) for n in (0, 1, 2, 3)]
    fr[0] = frame(np.zeros((0, NJ, 3), F32), np.zeros((0, 3), F32), np.zeros((0, 3), F32), sz(0))
    fr.append(frame(*crowd(rs, n_big, dup=0.2), (1080, 1920)))
    fr.append(frame(*far_outlier(rs, 4e4), (1920, 1080)))
    fr.append(frame(*far_outlier(rs, 1e3, n_in=9), (37, 53)))
    fr.append(frame(*ties_and_scales(rs), (2, 301)))
    fr.append(frame(*tuned_inlier(rs), (1080, 1920)))
    assert len(fr) == TUNED + 1
    j, c, t = crowd(rs, 6, dup=0.0)
    t[:, 2] = [1e-3, -2.0, 0.5, 3.0, -1e-4, 1e-6]             # pz near 0 and negative: large, far-off pixels
    fr.append(frame(j, c, t, (1, 1)))
    k = 10
    while len(fr) < 32:
        fr.append(frame(*crowd(rs, int(rs.randint(4, 40))), sz(k)))
        k += 1
    return fr


def layout(frames, cap):
    rows = sum(len(f["cam"]) for f in frames)
    assert rows <= cap
    joints, cam, ct = np.zeros((cap, NJ, 3), F32), np.zeros((cap, 3), F32), np.zeros((cap, 3), F32)
    bi = np.full(cap, len(frames), np.int64)
    o, starts = 0, []
    for b, f in enumerate(frames):
        n = len(f["cam"])
        starts.append(o)
        joints[o:o + n], cam[o:o + n], ct[o:o + n], bi[o:o + n] = f["joints"], f["cam"], f["ct"], b
        o += n
    pad = np.array([pad_row(*f["hw"]) for f in frames], F32)
    return dict(joints=joints, cam=cam, ct=ct, bi=bi, pad=pad, starts=starts, rows=rows)


def run_post(L, cap, count, nms, shared=None):
    """b200romp_bev_post_frames (shared None) or b200romp_bev_post with shared = (offsets6, img_max_side)."""
    lib = _lib.load()
    z = lambda *s, dt=torch.float32: torch.full(s, SENT, dtype=dt, device="cuda")
    o = dict(pj=z(cap, NJ, 2), keep=z(cap, dt=torch.int32), sel=z(cap, dt=torch.int32), n=z(1, dt=torch.int32))
    j, c, t, bi, pad = dev(L["joints"]), dev(L["cam"]), dev(L["ct"]), dev(L["bi"]), dev(L["pad"])
    betas, verts = torch.zeros(cap, 11, device="cuda"), torch.zeros(1, device="cuda")
    cnt = torch.tensor([count], dtype=torch.int32, device="cuda")
    B = len(L["pad"])
    head = (P(betas), None, None, P(verts), P(j), P(c), P(t), P(bi), B, cap, P(cnt))
    tail = (P(o["pj"]), P(o["keep"]), P(o["sel"]), P(o["n"]), stream())
    if shared is None:
        rc = lib.b200romp_bev_post_frames(*head, P(pad), float(nms), REL_T, *tail)
    else:
        off = (C.c_float * 6)(*[float(v) for v in shared[0]])
        rc = lib.b200romp_bev_post(*head, off, float(nms), REL_T, float(shared[1]), *tail)
    _lib.check(rc, "bev_post")
    torch.cuda.synchronize()
    return {k: v.cpu().numpy() for k, v in o.items()}


def frame_cap(L):
    """rows per frame the post-filter reads: 128 when the capacity exceeds 64 per frame (video mode), else 64."""
    return 128 if len(L["cam"]) > 64 * len(L["pad"]) else 64


def check_post(name, L, got, count, nms, shared=None, controls=()):
    """pj2d_org against float64, the kept rows of every frame against the enumerated float64 pipeline, the tails."""
    errs, bnds, n_amb = [], [], 0
    kept_all = []
    for b, st in enumerate(L["starts"]):
        n = sum(1 for i in range(st, count) if L["bi"][i] == b)
        if n == 0:
            continue
        n = min(n, frame_cap(L))
        r = slice(st, st + n)
        row = L["pad"][b] if shared is None else np.asarray(shared[0], F32)
        size = max(row[4], row[5])
        ref, bnd = project64(L["joints"][r], L["ct"][r], size, row[2], row[0])
        errs.append(np.abs(got["pj"][r] - ref).ravel()); bnds.append(bnd.ravel())
        thr = thr_px(nms, max(row[4], row[5]) if shared is None else shared[1])
        conf = -np.arange(n, dtype=F32)        # not read by the scale-based rule; the swapped-rule mutant reads it
        args = (got["pj"][r], L["cam"][r], L["ct"][r], conf, False, thr, REL_T, 0.25)
        sets = frame_sets(*args)
        kept = tuple(np.flatnonzero(got["keep"][r]).tolist())
        assert kept in sets, f"{name} frame {b}: kept {kept} not among float64's {sorted(sets)[:4]}"
        n_amb += len(sets) > 1
        for mut in controls:
            if kept not in frame_sets(*args, mutate=mut):
                controls = tuple(m for m in controls if m != mut)
        kept_all += [st + i for i in kept]
    accepted(f"{name} pj2d_org", np.concatenate(errs), np.concatenate(bnds))
    assert controls == (), f"{name}: controls {controls} not rejected"
    k = int(got["n"][0])
    assert k == len(kept_all) and got["sel"][:k].tolist() == kept_all, f"{name}: sel"
    assert (got["sel"][k:] == SENT).all() and (got["pj"][count:] == SENT).all(), f"{name}: a row past the count was written"
    assert (got["keep"][count:] == 0).all()
    print(f"{name}: {count} rows, {k} kept, {n_amb} frames with ambiguous decisions")


def emulate_post(L, count, nms, shared=None, formula="maxskip"):
    """the kernels' fp32 arithmetic on the CPU, in the layout run_post returns."""
    cap = len(L["cam"])
    got = dict(pj=np.full((cap, NJ, 2), SENT, F32), keep=np.zeros(cap, np.int32), sel=np.full(cap, SENT, np.int32),
               n=np.zeros(1, np.int32))
    kept_all, means = [], []
    for b, st in enumerate(L["starts"]):
        n = min(sum(1 for i in range(st, count) if L["bi"][i] == b), frame_cap(L))
        if n == 0:
            continue
        r = slice(st, st + n)
        row = L["pad"][b] if shared is None else np.asarray(shared[0], F32)
        got["pj"][r] = project32(L["joints"][r], L["ct"][r], max(row[4], row[5]), row[2], row[0])
        thr = thr_px(nms, max(row[4], row[5]) if shared is None else shared[1])
        k, m = frame_emulate32(got["pj"][r], L["cam"][r], L["ct"][r], None, False, thr, REL_T, 0.25, formula=formula)
        got["keep"][[st + i for i in k]] = 1
        kept_all += [st + i for i in k]
        means.append(m)
    got["sel"][:len(kept_all)] = kept_all
    got["n"][0] = len(kept_all)
    return got, means


def placement_layout(sizes, reps=3):
    return layout([frame(*placement_pool(), hw) for hw in sizes for _ in range(reps)], 2048)


def place(L8, pj, thr_of):
    """from each frame of the pool, the pair whose distance lands on the float below the frame's threshold (frames 3k),
    on it (3k+1) or on the float above (3k+2) -> (layout of the pairs, targets)."""
    frames, targets = [], []
    for b, st in enumerate(L8["starts"]):
        thr = F32(thr_of(b))
        t = [np.nextafter(thr, F32(0)), thr, np.nextafter(thr, F32(np.inf))][b % 3]
        for k in range(1, 8):
            m = place_scale(pj[[st, st + k]], t)
            if m is not None:
                break
        assert m is not None, "no pair of the pool places the distance"
        cam = L8["cam"][[st, st + k]].copy()
        cam[:, 0] = m / F32(2)
        frames.append(frame(L8["joints"][[st, st + k]], cam, L8["ct"][[st, st + k]], tuple(int(v) for v in L8["pad"][b][4:])))
        targets.append(t)
    return layout(frames, 2048), targets


def placement_misses(L, got, targets, thr_of, mutate=None):
    """frames whose kept rows differ from the exact decision t < thr (t <= thr for the mutant 'le')."""
    miss = []
    for b, st in enumerate(L["starts"]):
        thr = thr_of(b, mutate)
        below = targets[b] <= thr if mutate == "le" else targets[b] < thr
        assert dn32_exact(got["pj"][st:st + 2], L["cam"][st, 0] * 2) == targets[b]
        if tuple(np.flatnonzero(got["keep"][st:st + 2])) != ((0,) if below else (0, 1)):
            miss.append(b)
    return miss


def placement_cases():
    """(nms, sizes of post_frames, shared max sides of post): the default 20, and 16.3 whose threshold on a 1079-pixel
    side differs between double and float arithmetic."""
    return [(20.0, SIZES, (1, 2, 640)), (16.3, SIZES + [(1079, 700)], (1, 1079))]


def run_placement(runner):
    """runner(L, nms, shared) -> got.  Returns the mutants the cases reject."""
    rejected_by = set()
    muts = ("le", "no3", "float_thr")
    for nms, sizes, sides in placement_cases():
        L8 = placement_layout(sizes)
        thr_of = lambda b, mut=None: thr_px(nms, max(L8["pad"][b][4], L8["pad"][b][5]), mut)
        L, targets = place(L8, runner(L8, nms, None)["pj"], thr_of)
        got = runner(L, nms, None)
        assert placement_misses(L, got, targets, thr_of) == [], f"post_frames nms {nms}: threshold decisions"
        rejected_by |= {m for m in muts if placement_misses(L, got, targets, thr_of, m)}
        for side in sides:
            sh = (pad_row(side, side), side)
            L8s = placement_layout([(side, side)])
            thr_s = lambda b, mut=None: thr_px(nms, side, mut)
            Ls, targets = place(L8s, runner(L8s, nms, sh)["pj"], thr_s)
            got = runner(Ls, nms, sh)
            assert placement_misses(Ls, got, targets, thr_s) == [], f"post nms {nms} side {side}: threshold decisions"
            rejected_by |= {m for m in muts if placement_misses(Ls, got, targets, thr_s, m)}
        print(f"threshold placed exactly, nms_thresh {nms}: sizes {sizes}, shared sides {sides}: every decision exact")
    return rejected_by


# ============================================================================================ long-image merge
def long_rows(seed, n=1407):
    """n persons on a grid of the 1080 x 3840 image (most survive the suppression), a tenth of them near-duplicates of
    their predecessor (one pair with tied conf), person 0 at depth 4e4."""
    rs = np.random.RandomState(seed)
    gx, gy = np.meshgrid(np.linspace(-0.97, 0.97, 67), np.linspace(-0.25, 0.25, 21))
    cam = np.stack([rs.uniform(0.05, 0.15, n), gy.ravel()[:n], gx.ravel()[:n]], 1).astype(F32)
    rs.shuffle(cam[1:])
    conf = rs.uniform(0.1, 0.9, n).astype(F32)
    for i in np.flatnonzero(rs.uniform(size=n) < 0.1)[2:]:
        cam[i] = cam[i - 1] * F32(1.0001)
    dups = [i for i in range(2, n) if np.array_equal(cam[i], cam[i - 1] * F32(1.0001))]
    conf[dups[0]] = conf[dups[0] - 1]
    cam[0] = [F32(-1.6886e-3), 0.35, 0.01]            # above the grid, clear of every pair test
    return body(rs, n, 0.2), cam, conf


def run_long(joints, cam, conf, count, cap=1408, nms=20.0, hw=(1080, 3840)):
    lib = _lib.load()
    pad_info = long_image_plan(hw[0], hw[1], 0.8)[2]
    z = lambda *s, dt=torch.float32: torch.full(s, SENT, dtype=dt, device="cuda")
    o = dict(ct=z(cap, 3), pj=z(cap, NJ, 2), removed=z(cap, dt=torch.int32), sel=z(cap, dt=torch.int32), n=z(1, dt=torch.int32))
    ws = torch.full((int(lib.b200romp_bev_long_merge_workspace_bytes(cap)) // 4,), SENT, dtype=torch.int32, device="cuda")
    pad = lambda a: np.concatenate([a, np.zeros((cap - len(a),) + a.shape[1:], a.dtype)])
    j, c, f = dev(pad(joints[:count])), dev(pad(cam[:count])), dev(pad(conf[:count]))
    cnt = torch.tensor([count], dtype=torch.int32, device="cuda")
    off = (C.c_float * 6)(*[float(v) for v in pad_info])
    _lib.check(lib.b200romp_bev_long_merge(P(c), P(j), P(f), cap, P(cnt), off, nms, REL_T, float(hw[1]), P(o["ct"]), P(o["pj"]),
                                           P(o["removed"]), P(ws), P(o["sel"]), P(o["n"]), stream()), "bev_long_merge")
    torch.cuda.synchronize()
    got = {k: v.cpu().numpy() for k, v in o.items()}
    w = ws.cpu().numpy()
    got["ws_nk"], got["ws_sel"], got["ws_mean"] = int(w[0]), w[4:4 + cap], w[4 + cap:4 + 2 * cap].view(F32)
    return got, pad_info


def check_long(name, joints, cam, conf, count, got, pad_info, nms=20.0, side=3840, dist=None, mean_formula_ok=True):
    """-> worst mean-distance ratio.  cam_trans, pj2d_org, survivors of the suppression, row means, kept rows, tails."""
    n = count
    ct, ct_b = cam_trans64(cam[:n])
    accepted(f"{name} cam_trans", np.abs(got["ct"][:n] - ct), ct_b)
    ref, bnd = project64(joints[:n], got["ct"][:n], max(pad_info[4], pad_info[5]), pad_info[2], pad_info[0])
    accepted(f"{name} pj2d_org", np.abs(got["pj"][:n] - ref), bnd)
    thr = thr_px(nms, side)
    nk = got["ws_nk"]
    sel1 = got["ws_sel"][:nk].tolist()
    assert got["removed"][:n].tolist() == [0 if i in set(sel1) else 1 for i in range(n)], f"{name}: removed flags"
    sets = frame_sets(got["pj"][:n], cam[:n], got["ct"][:n], conf[:n], True, thr, REL_T, 0.5, dist=dist)
    k = int(got["n"][0])
    kept = tuple(got["sel"][:k].tolist())
    assert kept in sets, f"{name}: kept rows not among float64's"
    ratio = 0.0
    if nk >= 3:
        mean, e_mean, _, _ = outlier_stats(got["ct"][sel1])
        ratio = report(f"{name} row means ({nk} survivors)", np.abs(got["ws_mean"][:nk] - mean), e_mean)
    assert (got["ws_mean"][nk:].view(np.int32) == SENT).all()
    assert (got["sel"][k:] == SENT).all() and (got["ct"][n:] == SENT).all() and (got["pj"][n:] == SENT).all()
    assert (got["removed"][n:] == SENT).all() and (got["ws_sel"][nk:] == SENT).all()
    print(f"{name}: {n} rows, {nk} after the suppression, {k} kept ({len(sets)} resolutions)")
    return ratio


# ================================================================================================ crop stage
CROP_ROWS = dict(verts=6890 * 3, joints=NJ * 3, thetas=72, betas=11, params_pred=146, conf=1)


def crop_frames(seed, h=1080, w=3840):
    """the crops of an h x w image (22 for 1080 x 3840), each with a few random persons (some near-duplicates, cam x inside
    both limits) and, on crops 0, 1, the middle one and the last, probes at every finite limit of the crop table and one
    float either side.  Probes have conf 0.95, cam[:,0] = 1 (never an outlier at scale_thresh 1) and pixels clear of
    everyone, so their fate is the boundary drop alone.  Crop 0 adds a dropped duplicate of a person with higher conf
    (it would suppress that person were it left in the filters), crop 1 a pair with tied conf, crop 2 a pair whose
    smaller scale has the higher conf, crop 3 a far person with scale 0.6 (an outlier at scale_thresh 1, not at 0.25)."""
    pad_length, boxes, _ = long_image_plan(h, w, 0.8)
    tab = long_image_crop_table(boxes, pad_length, h, w, 20.0)
    rs = np.random.RandomState(seed)
    K = len(boxes)
    out = []
    at = lambda a, b, z: np.array([a * z, b * z, z], F32)
    for c in range(K):
        n = int(rs.randint(3, 12))
        joints, cam, ct = crowd(rs, n, dup=0.25)
        cam[:, 0] = rs.uniform(0.3, 0.9, n)
        cam[:, 2] = rs.uniform(-0.5, 0.5, n)
        conf = rs.uniform(0.1, 0.9, n).astype(F32)
        extra, probes = [], []
        if c in (0, 1, K // 2, K - 1):
            k = 0
            for lim in tab[c, :2]:
                if not np.isfinite(lim):
                    continue
                for x, kind in ((np.nextafter(lim, F32(-np.inf)), "below"), (lim, "at"), (np.nextafter(lim, F32(np.inf)), "above")):
                    extra.append((at(-0.6 + 0.2 * k, 0.45, 6.0), [1.0, 0.0, x], 0.95))
                    probes.append((n + len(extra) - 1, lim == tab[c, 0], kind))
                    k += 1
        if c == 0:
            q = at(0.3, -0.45, 5.0)
            extra.append((q, [1.0, 0.0, 0.0], 0.5))
            extra.append((q, [1.0, 0.0, np.nextafter(tab[c, 0], F32(np.inf))], 0.97))
        if c == 1:
            q = at(-0.3, -0.45, 5.0)
            extra += [(q, [1.0, 0.0, 0.0], 0.6), (q, [1.0, 0.0, 0.1], 0.6)]
        if c == 2:
            q = at(0.0, -0.45, 5.0)
            extra += [(q, [0.95, 0.0, 0.0], 0.7), (q, [1.0, 0.0, 0.1], 0.6)]
        if c == 3:
            extra.append((at(-0.3, -0.6, 200.0), [0.6, 0.0, 0.0], 0.5))
        if extra:
            same = body(rs, 1)[0]
            joints = np.concatenate([joints, np.repeat(same[None], len(extra), 0)])
            ct = np.concatenate([ct, np.stack([e[0] for e in extra])])
            cam = np.concatenate([cam, np.array([e[1] for e in extra], F32)])
            conf = np.concatenate([conf, np.array([e[2] for e in extra], F32)])
        m = len(cam)
        out.append(dict(joints=joints, cam=cam.astype(F32), ct=ct.astype(F32), conf=conf, tab=tab[c], probes=probes,
                        verts=rs.normal(0, 1, (m, CROP_ROWS["verts"])).astype(F32),
                        thetas=rs.normal(0, 1, (m, 72)).astype(F32), betas=rs.normal(0, 1, (m, 11)).astype(F32),
                        params_pred=rs.normal(0, 1, (m, 146)).astype(F32)))
    return out, tab


def crop_chunk(frames):
    """rows of one chunk of crops, grouped by frame."""
    cat = lambda k: np.concatenate([f[k] for f in frames])
    d = {k: cat(k) for k in ("joints", "cam", "ct", "conf", "verts", "thetas", "betas", "params_pred")}
    d["bi"] = np.concatenate([np.full(len(f["cam"]), b, np.int64) for b, f in enumerate(frames)])
    d["starts"] = np.cumsum([0] + [len(f["cam"]) for f in frames])[:-1].tolist()
    return d


def cam_full32(cam, tab):
    """convert_crop_cam_params2full_image: cam *= scale, cam[:,2] += shift, in place in fp32."""
    c = (cam * tab[4]).astype(F32)
    c[:, 2] = c[:, 2] + tab[5]
    return c


def crop_drop(cam, tab):
    x = cam[:, 2]
    return (x > tab[0]) | (x < tab[1])


def run_crop(frames_all, tab, chunk, acc_capacity):
    """b200romp_bev_crop_post over the image's crops in chunks of `chunk` -> (per-chunk outputs, accumulated rows)."""
    lib = _lib.load()
    z = lambda *s, dt=torch.float32: torch.full(s, SENT, dtype=dt, device="cuda")
    acc = {k: z(acc_capacity, w) for k, w in CROP_ROWS.items()}
    acc["cam"] = z(acc_capacity, 3)
    acc_count = torch.zeros(2, dtype=torch.int32, device="cuda")
    ctl = torch.zeros(2, dtype=torch.int32, device="cuda")
    tab_d = dev(tab)
    chunks = []
    for c0 in range(0, len(frames_all), chunk):
        fr = frames_all[c0:c0 + chunk]
        nb, d = len(fr), crop_chunk(fr)
        cap, rows = nb * 64, len(d["cam"])
        pad = lambda a: np.concatenate([a, np.zeros((cap - len(a),) + a.shape[1:], a.dtype)])
        bi = np.concatenate([d["bi"], np.full(cap - rows, nb, np.int64)])
        t = {k: dev(pad(d[k])) for k in ("joints", "cam", "ct", "conf", "verts", "thetas", "betas", "params_pred")}
        o = dict(pj=z(cap, NJ, 2), keep=z(cap, dt=torch.int32), sel=z(cap, dt=torch.int32), cam_full=z(cap, 3))
        cnt = torch.tensor([rows], dtype=torch.int32, device="cuda")
        _lib.check(lib.b200romp_bev_crop_post(
            P(t["betas"]), None, None, P(t["verts"]), P(t["joints"]), P(t["thetas"]), P(t["params_pred"]), P(t["conf"]),
            P(t["cam"]), P(t["ct"]), P(dev(bi)), nb, cap, P(cnt), P(tab_d), c0, REL_T, P(o["pj"]), P(o["keep"]), P(o["sel"]),
            P(o["cam_full"]), acc_capacity, P(acc_count), P(ctl), P(acc["verts"]), P(acc["joints"]), P(acc["thetas"]),
            P(acc["betas"]), P(acc["params_pred"]), P(acc["conf"]), P(acc["cam"]), stream()), "bev_crop_post")
        torch.cuda.synchronize()
        chunks.append((c0, d, {k: v.cpu().numpy() for k, v in o.items()}))
    return chunks, {k: v.cpu().numpy() for k, v in acc.items()}, acc_count.cpu().numpy()


def check_crop_frames(name, frames, tab, c0, d, got, controls):
    """pj2d, cam_full, the boundary probes and the kept rows of each crop of one chunk; returns the controls not yet
    rejected."""
    errs, bnds = [], []
    for b, st in enumerate(d["starts"]):
        f, c = frames[b], c0 + b
        n = len(f["cam"])
        r = slice(st, st + n)
        ref, bnd = project64(f["joints"], f["ct"], tab[c, 2], 0.0, 0.0)
        errs.append(np.abs(got["pj"][r] - ref).ravel()); bnds.append(bnd.ravel())
        assert got["cam_full"][r].tobytes() == cam_full32(f["cam"], tab[c]).tobytes(), f"{name} crop {c}: cam_full"
        drop = crop_drop(f["cam"], tab[c])
        keep = got["keep"][r]
        for i, left_limit, kind in f["probes"]:
            dropped = kind == "above" if left_limit else kind == "below"
            assert keep[i] == (0 if dropped else 1), f"{name} crop {c}: probe {kind} the {'left' if left_limit else 'right'} limit"
        args = (got["pj"][r], f["cam"], f["ct"], f["conf"], True, F64(tab[c, 3]), REL_T, 1.0, drop)
        kept = tuple(np.flatnonzero(keep).tolist())
        assert kept in frame_sets(*args), f"{name} crop {c}: kept {kept} not among float64's"
        controls = tuple(m for m in controls if kept in frame_sets(*args, mutate=m))
    accepted(f"{name} pj2d", np.concatenate(errs), np.concatenate(bnds))
    return controls


def check_crop(name, frames_all, tab, chunks, acc, acc_count, acc_capacity):
    controls = ("keep_dropped", "tie_reversed", "swap_rules", "scale_quarter")
    want = {k: [] for k in list(CROP_ROWS) + ["cam"]}
    total = 0
    for c0, d, got in chunks:
        frames = frames_all[c0:c0 + len(d["starts"])]
        controls = check_crop_frames(name, frames, tab, c0, d, got, controls)
        rows = len(d["cam"])
        total += rows
        assert (got["pj"][rows:] == SENT).all() and (got["cam_full"][rows:] == SENT).all() and (got["keep"][rows:] == 0).all()
        sel = np.flatnonzero(got["keep"][:rows])
        for k in CROP_ROWS:
            want[k].append(d[k][sel].reshape(len(sel), -1))
        want["cam"].append(got["cam_full"][sel])
    assert controls == (), f"{name}: controls {controls} not rejected"
    kept = sum(len(w) for w in want["cam"])
    k0 = min(kept, acc_capacity)
    assert acc_count.tolist() == [k0, total], f"{name}: acc_count {acc_count.tolist()} != {[k0, total]}"
    for k, parts in want.items():
        w = np.concatenate(parts)[:k0]
        a = acc[k].reshape(acc_capacity, -1)
        assert a[:k0].tobytes() == w.tobytes(), f"{name}: appended {k} rows"
        assert (a[k0:] == SENT).all(), f"{name}: {k} rows past the count"
    print(f"{name}: {total} persons in {len(frames_all)} crops, {kept} survivors, {k0} appended; controls rejected")
    return kept


def emulate_crop(frames_all, tab, chunk, acc_capacity):
    """the crop stage's fp32 arithmetic on the CPU, in run_crop's layout."""
    chunks, want = [], {k: [] for k in list(CROP_ROWS) + ["cam"]}
    total = 0
    for c0 in range(0, len(frames_all), chunk):
        fr = frames_all[c0:c0 + chunk]
        d = crop_chunk(fr)
        cap, rows = len(fr) * 64, len(d["cam"])
        got = dict(pj=np.full((cap, NJ, 2), SENT, F32), keep=np.zeros(cap, np.int32), cam_full=np.full((cap, 3), SENT, F32))
        for b, st in enumerate(d["starts"]):
            f, c = fr[b], c0 + b
            r = slice(st, st + len(f["cam"]))
            got["pj"][r] = project32(f["joints"], f["ct"], tab[c, 2], 0.0, 0.0)
            got["cam_full"][r] = cam_full32(f["cam"], tab[c])
            k, _ = frame_emulate32(got["pj"][r], f["cam"], f["ct"], f["conf"], True, tab[c, 3], REL_T, 1.0, crop_drop(f["cam"], tab[c]))
            got["keep"][[st + i for i in k]] = 1
        sel = np.flatnonzero(got["keep"][:rows])
        for k in CROP_ROWS:
            want[k].append(d[k][sel].reshape(len(sel), -1))
        want["cam"].append(got["cam_full"][sel])
        total += rows
        chunks.append((c0, d, got))
    kept = sum(len(w) for w in want["cam"])
    k0 = min(kept, acc_capacity)
    acc = {}
    for k, parts in want.items():
        a = np.full((acc_capacity, np.concatenate(parts).shape[1]), SENT, F32)
        a[:k0] = np.concatenate(parts)[:k0]
        acc[k] = a
    return chunks, acc, np.array([k0, total], np.int32)


# ================================================================================================== GPU tests
@gpu
def test_threshold_placed_exactly():
    rej = run_placement(lambda L, nms, sh: run_post(L, 2048, L["rows"], nms, sh))
    assert rej == {"le", "no3", "float_thr"}, f"controls not rejected: {({'le', 'no3', 'float_thr'} - rej)}"
    print("  controls rejected: <= for <, max(h, w) for max(h, w, 3), the threshold formed in float")


@gpu
def test_post_frames_cap64():
    fr = post_frames(1)
    L = layout(fr, 2048)
    rows = L["rows"]
    got = run_post(L, 2048, rows, 20.0)
    check_post("post_frames CAP 64", L, got, rows, 20.0, controls=("tie_reversed", "swap_rules"))
    r = slice(L["starts"][TUNED], L["starts"][TUNED] + len(fr[TUNED]["cam"]))
    margin = tuned_margin(got["pj"][r], L["cam"][r], L["ct"][r], thr_px(20.0, 1920))
    print(f"tuned inlier: |rel - thr| = {margin:.2f} of its fp32 bound, every person of its frame reaches remove_outlier")
    assert margin <= 1.0
    part = run_post(L, 2048, rows - 30, 20.0)
    check_post("post_frames, device count 30 below the rows", L, part, rows - 30, 20.0)
    for b, f in enumerate(fr):
        h, w = f["hw"]
        one = run_post(L, 2048, rows, 20.0, (L["pad"][b], max(h, w)))
        st, n = L["starts"][b], len(f["cam"])
        assert one["pj"][st:st + n].tobytes() == got["pj"][st:st + n].tobytes(), f"frame {b}: pj2d_org of _post"
        assert one["keep"][st:st + n].tobytes() == got["keep"][st:st + n].tobytes(), f"frame {b}: keep of _post"
    print("post per frame bit-equal to post_frames")


@gpu
def test_post_frames_cap128():
    rs = np.random.RandomState(7)
    fr = [frame(*crowd(rs, 128, dup=0.2), (1080, 1920)), frame(*far_outlier(rs, 4e4, n_in=100), (1920, 1080)),
          frame(*crowd(rs, 3), (2, 2)), frame(np.zeros((0, NJ, 3), F32), np.zeros((0, 3), F32), np.zeros((0, 3), F32), (1, 1))]
    L = layout(fr, 2 * 4 * 64)
    got = run_post(L, 512, L["rows"], 20.0)
    check_post("post_frames CAP 128", L, got, L["rows"], 20.0)
    assert got["keep"][64:128].any()                # the rows past 64 of a frame take part


@gpu
def test_long_merge():
    joints, cam, conf = long_rows(3)
    ratios, dist = [], None
    full, pad_info = run_long(joints, cam, conf, 1407)
    dist = dn_matrix(full["pj"][:1407])
    for n in (0, 1, 2, 3, 15, 16, 17, 1023, 1024, 1025, 1407):
        got, _ = run_long(joints, cam, conf, n) if n != 1407 else (full, pad_info)
        if n:
            assert got["pj"][:n].tobytes() == full["pj"][:n].tobytes()
        ratios.append(check_long(f"long_merge count {n}", joints, cam, conf, n, got, pad_info, dist=dist[:n, :n]))
    assert full["ws_nk"] > 1024 and int(full["n"][0]) > 128
    assert max(ratios) <= 1.0, "row means of remove_outlier outside the bound of the sorted-row formula"


@gpu
def test_gather_rows():
    lib = _lib.load()
    rs = np.random.RandomState(11)
    for row_bytes in (4, 8, 12, 584, 82680):
        cap = 300
        words = row_bytes // 4
        src = dev(rs.randint(-2 ** 31, 2 ** 31, (cap, words)).astype(np.int32))
        for n in (0, 17, cap):
            sel = np.full(cap, SENT, np.int32)
            sel[:n] = rs.permutation(cap)[:n]
            dst = torch.full((cap, words), SENT, dtype=torch.int32, device="cuda")
            cnt = torch.tensor([n], dtype=torch.int32, device="cuda")
            _lib.check(lib.b200romp_gather_rows(P(src), row_bytes, P(dev(sel)), P(cnt), cap, P(dst), stream()), "gather_rows")
            torch.cuda.synchronize()
            d, s = dst.cpu().numpy(), src.cpu().numpy()
            assert d[:n].tobytes() == s[sel[:n]].tobytes() and (d[n:] == SENT).all(), f"gather_rows {row_bytes} B, {n} rows"
    print("gather_rows: rows of 4, 8, 12, 584 and 82680 bytes, counts 0, 17 and capacity, in arbitrary order")


@gpu
def test_crop_post():
    frames, tab = crop_frames(1)
    K = len(frames)
    full = run_crop(frames, tab, 12, K * 64)
    kept = check_crop("crop_post, 2 chunks", frames, tab, *full, K * 64)
    k1 = int(full[0][0][2]["keep"].sum())
    assert 0 < k1 and k1 + 3 < kept
    cut = run_crop(frames, tab, 12, k1 + 3)
    check_crop(f"crop_post, acc_capacity {k1 + 3} cuts the second chunk", frames, tab, *cut, k1 + 3)


# ================================================================================================== CPU tests
def test_threshold_numbers_cpu():
    assert thr_px(20.0, 1) == 0.09375 and thr_px(20.0, 1, "no3") == 0.03125 and thr_px(20.0, 2) == 0.09375
    assert F32(thr_px(16.3, 1079)) == F32(27.480782) and thr_px(16.3, 1079) != thr_px(16.3, 1079, "float_thr")
    assert thr_px(20.0, 1080) == thr_px(20.0, 1080, "float_thr") == 33.75


def test_placement_emulated_cpu():
    """the exact placement with the kernel's fp32 arithmetic emulated: every decision exact, every mutant rejected."""
    rej = run_placement(lambda L, nms, sh: emulate_post(L, L["rows"], nms, sh)[0])
    assert rej == {"le", "no3", "float_thr"}


def test_post_emulated_cpu():
    """post_frames' batch through the checks with the fp32 emulation: the kept rows are among float64's, the mutants of
    the tie and scale/conf rules are rejected."""
    L = layout(post_frames(1), 2048)
    got, _ = emulate_post(L, L["rows"], 20.0)
    check_post("emulated post CAP 64", L, got, L["rows"], 20.0, controls=("tie_reversed", "swap_rules"))


def test_row_mean_formulas_cpu():
    """the reference's sorted-row mean and the kernels' max-skipping sum pass the mean check; (sum - min - max), which
    the kernels computed before, fails it on a far outlier (depth 1e3 and 4e4)."""
    rs = np.random.RandomState(5)
    for depth in (1e3, 4e4):
        ct = far_outlier(rs, depth)[2]
        mean, e_mean, _, _ = outlier_stats(ct)
        accepted(f"sorted-row fp32 mean, outlier at depth {depth:g}", np.abs(row_means32(ct, "sort") - mean), e_mean)
        accepted(f"max-skipping fp32 mean, outlier at depth {depth:g}", np.abs(row_means32(ct, "maxskip") - mean), e_mean)
        rejected(f"(sum - min - max) fp32 mean, outlier at depth {depth:g}", np.abs(row_means32(ct, "summinmax") - mean), e_mean)
    joints, cam, conf = long_rows(3, 200)
    ct = cam_trans32(cam)
    mean, e_mean, _, _ = outlier_stats(ct)
    accepted("max-skipping fp32 mean, 200 persons", np.abs(row_means32(ct, "maxskip") - mean), e_mean)


def test_tuned_inlier_cpu():
    """the tuned inlier lies inside its fp32 bound on the rows that reach remove_outlier; (sum - min - max) moves its rel
    by a small fraction of that bound only, so on this frame the formula the kernels used before cannot flip the decision
    beyond what a correct fp32 evaluation may do: only the row-mean check (above) tells the two apart."""
    L = layout(post_frames(1), 2048)
    got, _ = emulate_post(L, L["rows"], 20.0)
    st, n = L["starts"][TUNED], int((L["bi"] == TUNED).sum())
    r = slice(st, st + n)
    ct = L["ct"][r]
    assert tuned_margin(got["pj"][r], L["cam"][r], ct, thr_px(20.0, 1920)) <= 1.0
    _, _, rel, e_rel = outlier_stats(ct)
    for formula in ("sort", "maxskip", "summinmax"):
        m = row_means32(ct, formula)
        tot = F32(0)
        for x in m:
            tot = F32(tot + x)
        rel32 = m / ((tot - m) / F32(n - 1))
        print(f"tuned inlier, {formula} fp32 rel: {abs(float(rel32[1]) - rel[1]) / e_rel[1]:.3f} of the bound")
        assert abs(float(rel32[1]) - rel[1]) <= e_rel[1]


def test_crop_emulated_cpu():
    """the crop stage's fp32 emulation through the GPU test's checks: accepted, and every control rejected."""
    frames, tab = crop_frames(1)
    K = len(frames)
    full = emulate_crop(frames, tab, 12, K * 64)
    kept = check_crop("emulated crop_post", frames, tab, *full, K * 64)
    k1 = int(full[0][0][2]["keep"].sum())
    cut = emulate_crop(frames, tab, 12, k1 + 3)
    check_crop("emulated crop_post, cut", frames, tab, *cut, k1 + 3)
    assert k1 + 3 < kept
