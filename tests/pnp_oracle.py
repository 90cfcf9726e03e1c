"""fp64 numpy restatement of the reference's default cam_trans (``estimate_translation``, simple_romp/romp/utils.py:391-436):
the validity mask of the 24 SMPL joints, then OpenCV's ``solvePnPRansac(EPnP, reprojectionError=20, iterationsCount=100)``
loop (RANSACPointSetRegistrator::run with OpenCV's RNG, 5-point subsets and RANSACUpdateNumIters) around the published
EPnP of Lepetit, Moreno-Noguer and Fua (IJCV 2009), the estimator of ``--cam_trans epnp`` (csrc/pnp.cu).

``kernel`` selects the 5-point solver: ``epnp`` (the published method, what the device runs) or ``cv2``
(``cv2.solvePnP(SOLVEPNP_EPNP)`` itself, to check the loop against ``cv2.solvePnPRansac``)."""
from __future__ import annotations

import math

import numpy as np

FOCAL, CENTER = 443.4, 256.0
THRESH2 = np.float32(20.0 * 20.0)
MODEL_POINTS, MAX_ITERS, CONFIDENCE = 5, 100, 0.99
INVALID = np.array([-1.0, -1.0, -1.0], np.float32)
K = np.array([[FOCAL, 0, CENTER], [0, FOCAL, CENTER], [0, 0, 1.0]])


def pj2d_valid(joints, cam):
    """utils.py:404-422: pj2d = (xy * s + t + 1) * 256 in float32 on the first 24 joints; joint i is valid when
    pj2d_y > -2 and z != -2.  Returns (j3 [n,24,3] f32, pj2d [n,24,2] f32, valid [n,24] bool)."""
    joints, cam = np.asarray(joints, np.float32), np.asarray(cam, np.float32)
    j3 = np.ascontiguousarray(joints[:, :24])
    p2 = (j3[:, :, :2] * cam[:, None, 0:1] + cam[:, None, 1:3] + np.float32(1.0)) * np.float32(256.0)
    return j3, p2, (p2[:, :, 1] > -2.0) & (j3[:, :, 2] != -2.0)


def cv_rng_subsets(n, count=MAX_ITERS):
    """OpenCV's RNG((uint64)-1) drawing ``count`` 5-index subsets of range(n) like RANSACPointSetRegistrator::getSubset:
    a draw equal to an earlier index of the same subset is drawn again; no subset is rejected."""
    state, out = 0xFFFFFFFFFFFFFFFF, []
    for _ in range(count):
        idx = []
        while len(idx) < MODEL_POINTS:
            state = ((state & 0xFFFFFFFF) * 4164903690 + (state >> 32)) & 0xFFFFFFFFFFFFFFFF
            v = (state & 0xFFFFFFFF) % n
            if v not in idx:
                idx.append(v)
        out.append(idx)
    return np.array(out, np.int64)


def ransac_update_num_iters(p, ep, model_points, max_iters):
    """cv::RANSACUpdateNumIters."""
    p, ep = min(max(p, 0.0), 1.0), min(max(ep, 0.0), 1.0)
    num = max(1.0 - p, np.finfo(np.float64).tiny)
    denom = 1.0 - math.pow(1.0 - ep, model_points)
    if denom < np.finfo(np.float64).tiny:
        return 0
    num, denom = math.log(num), math.log(denom)
    if denom >= 0 or -num >= max_iters * (-denom):
        return max_iters
    return int(np.rint(num / denom))       # cvRound: nearest, ties to even


def normalized_pixels(p2, hypothesis):
    """The pixels EPnP sees.  cv2 undistorts to normalised coordinates of the input's type and multiplies back: the
    hypotheses' subsets are float32 (solvePnPRansac converts its input to float32), the final fit is float64."""
    x = (np.asarray(p2, np.float64) - CENTER) * (1.0 / FOCAL)
    if hypothesis:
        x = x.astype(np.float32).astype(np.float64)
    return x * FOCAL + CENTER


def _lstsq(A, b):
    return np.linalg.lstsq(A, b, rcond=None)[0]


def opencv_svd_rows(a):
    """cvSVD of a symmetric 3x3 (JacobiSVDImpl_: one-sided Jacobi on the rows of Aᵀ, eps = 10 DBL_EPSILON, rows sorted
    by norm and normalised) -> (singular values descending, rows).  EPnP's control points lie along these rows, and with
    noisy points the pose depends on the sign of each: this is the rule that gives OpenCV's signs."""
    At, eps = np.array(a, np.float64).T.copy(), 10.0 * np.finfo(np.float64).eps
    W = (At * At).sum(1)
    for _ in range(30):
        changed = False
        for i, j in ((0, 1), (0, 2), (1, 2)):
            p = float(At[i] @ At[j])
            if abs(p) <= eps * math.sqrt(W[i] * W[j]):
                continue
            p *= 2.0
            beta = W[i] - W[j]
            gamma = math.hypot(p, beta)
            if beta < 0:
                s = math.sqrt((gamma - beta) * 0.5 / gamma)
                c = p / (gamma * s * 2.0)
            else:
                c = math.sqrt((gamma + beta) / (gamma * 2.0))
                s = p / (gamma * c * 2.0)
            At[i], At[j] = c * At[i] + s * At[j], -s * At[i] + c * At[j]
            W[i], W[j] = At[i] @ At[i], At[j] @ At[j]
            changed = True
        if not changed:
            break
    W = np.sqrt((At * At).sum(1))
    o = [0, 1, 2]
    for i in range(2):
        j = i
        for k in range(i + 1, 3):
            if W[o[j]] < W[o[k]]:
                j = k
        o[i], o[j] = o[j], o[i]
    return W[o], np.array([At[k] / W[k] if W[k] > 0 else At[k] * 0.0 for k in o])


def epnp(pws, us):
    """The published EPnP in fp64: control points at the centroid plus the principal axes (signed as OpenCV signs them,
    opencv_svd_rows) scaled by sqrt(eigenvalue / n),
    the four smallest eigenvectors of MᵀM, the three beta approximations each refined by 5 Gauss-Newton steps on the
    six control-point distances, and the candidate with the smallest mean reprojection error.  With fewer than 6 points
    the exact null space of MᵀM gets a fixed basis (the eigenvectors of diag(1..12) restricted to it), which the
    published method leaves to the eigen-solver.  Returns (R, t)."""
    pws, us = np.asarray(pws, np.float64), np.asarray(us, np.float64)
    n = len(pws)
    c0 = pws.mean(0)
    w, uc = opencv_svd_rows((pws - c0).T @ (pws - c0))
    cws = np.vstack([c0] + [c0 + math.sqrt(max(w[k], 0.0) / n) * uc[k] for k in range(3)])
    al = np.empty((n, 4))
    al[:, 1:] = (pws - c0) @ np.linalg.inv((cws[1:] - c0).T).T
    al[:, 0] = 1.0 - al[:, 1:].sum(1)
    M = np.zeros((2 * n, 12))
    M[0::2, 0::3] = al * FOCAL
    M[0::2, 2::3] = al * (CENTER - us[:, 0:1])
    M[1::2, 1::3] = al * FOCAL
    M[1::2, 2::3] = al * (CENTER - us[:, 1:2])
    ew, ev = np.linalg.eigh(M.T @ M)
    nv = ev[:, np.argsort(ew)[:4]]                      # column 0: smallest eigenvalue
    d = 12 - 2 * n
    if d > 0:   # exact null space (n = 5: 2 dims, n = 4: 4): its basis fixed as in csrc/pnp.cu null_space_basis
        bw, be = np.linalg.eigh(nv[:, :d].T @ (np.arange(1, 13)[:, None] * nv[:, :d]))
        nv[:, :d] = nv[:, :d] @ be[:, np.argsort(bw)]
    nv = [nv[:, k] for k in range(4)]
    pairs = [(0, 1), (0, 2), (0, 3), (1, 2), (1, 3), (2, 3)]
    dv = [[x[3 * a:3 * a + 3] - x[3 * b:3 * b + 3] for a, b in pairs] for x in nv]
    L = np.array([[dv[0][i] @ dv[0][i], 2 * dv[0][i] @ dv[1][i], dv[1][i] @ dv[1][i], 2 * dv[0][i] @ dv[2][i],
                   2 * dv[1][i] @ dv[2][i], dv[2][i] @ dv[2][i], 2 * dv[0][i] @ dv[3][i], 2 * dv[1][i] @ dv[3][i],
                   2 * dv[2][i] @ dv[3][i], dv[3][i] @ dv[3][i]] for i in range(6)])
    rho = np.array([np.sum((cws[a] - cws[b]) ** 2) for a, b in pairs])

    def gauss_newton(B):
        for _ in range(5):
            A = np.stack([2 * L[:, 0] * B[0] + L[:, 1] * B[1] + L[:, 3] * B[2] + L[:, 6] * B[3],
                          L[:, 1] * B[0] + 2 * L[:, 2] * B[1] + L[:, 4] * B[2] + L[:, 7] * B[3],
                          L[:, 3] * B[0] + L[:, 4] * B[1] + 2 * L[:, 5] * B[2] + L[:, 8] * B[3],
                          L[:, 6] * B[0] + L[:, 7] * B[1] + L[:, 8] * B[2] + 2 * L[:, 9] * B[3]], 1)
            q = np.array([B[0] * B[0], B[0] * B[1], B[1] * B[1], B[0] * B[2], B[1] * B[2], B[2] * B[2], B[0] * B[3],
                          B[1] * B[3], B[2] * B[3], B[3] * B[3]])
            B = B + _lstsq(A, rho - L @ q)
        return B

    def first_two(b):
        if b[0] < 0:
            b0, b1 = math.sqrt(-b[0]), (math.sqrt(-b[2]) if b[2] < 0 else 0.0)
        else:
            b0, b1 = math.sqrt(b[0]), (math.sqrt(b[2]) if b[2] > 0 else 0.0)
        return (-b0 if b[1] < 0 else b0), b1

    b4 = _lstsq(L[:, [0, 1, 3, 6]], rho)
    b0 = math.sqrt(abs(b4[0]))
    s = -1.0 if b4[0] < 0 else 1.0
    cands = [np.array([b0, s * b4[1] / b0, s * b4[2] / b0, s * b4[3] / b0])]
    cands.append(np.array([*first_two(_lstsq(L[:, :3], rho)), 0.0, 0.0]))
    b5 = _lstsq(L[:, :5], rho)
    f0, f1 = first_two(b5)
    cands.append(np.array([f0, f1, b5[3] / f0, 0.0]))

    best = None
    for B in cands:
        B = gauss_newton(B)
        ccs = sum(B[i] * nv[i] for i in range(4)).reshape(4, 3)
        pcs = al @ ccs
        if pcs[0, 2] < 0:
            pcs = -pcs
        pc0, pw0 = pcs.mean(0), pws.mean(0)
        U, _, Vt = np.linalg.svd((pcs - pc0).T @ (pws - pw0))
        R = U @ Vt
        if np.linalg.det(R) < 0:
            R[2] = -R[2]
        t = pc0 - R @ pw0
        X = pws @ R.T + t
        err = np.mean(np.hypot(us[:, 0] - (CENTER + FOCAL * X[:, 0] / X[:, 2]), us[:, 1] - (CENTER + FOCAL * X[:, 1] / X[:, 2])))
        if best is None or err < best[0]:
            best = (err, R, t)
    return best[1], best[2]


def cv2_epnp(pws, p2_f32, hypothesis):
    """cv2.solvePnP(SOLVEPNP_EPNP) as the kernel, on float32 points for a hypothesis and float64 for the final fit."""
    import cv2
    dt = np.float32 if hypothesis else np.float64
    _, rvec, tvec = cv2.solvePnP(np.asarray(pws, dt), np.asarray(p2_f32, dt), K, None, flags=cv2.SOLVEPNP_EPNP)
    return cv2.Rodrigues(rvec)[0], tvec[:, 0]


def _solve(kernel, pws, p2, hypothesis):
    if kernel == "cv2":
        return cv2_epnp(pws, p2, hypothesis)
    return epnp(pws, normalized_pixels(p2, hypothesis))


def _subset(kernel, idx):
    """cv2 receives a subset in draw order; the device reads it in joint order (the same points, summed in another order)."""
    return idx if kernel == "cv2" else np.sort(idx)


def reprojection_errors(R, t, pws, p2):
    """findInliers' error: the projection in double rounded to float32, then dx*dx + dy*dy in float32."""
    X = np.asarray(pws, np.float64) @ R.T + t
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        iz = 1.0 / X[:, 2]
        proj = np.stack([X[:, 0] * iz * FOCAL + CENTER, X[:, 1] * iz * FOCAL + CENTER], 1).astype(np.float32)
        d = np.asarray(p2, np.float32) - proj
        return d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]


def ransac_one(pws, p2, kernel="epnp"):
    """One person's valid joints (float32 [n,3], [n,2]) -> (tvec float64 [3] or None, inlier bool [n], closest |err-400|
    of any joint in any evaluated hypothesis)."""
    n = len(pws)
    if n < 4:
        return None, np.zeros(n, bool), np.inf
    if n <= MODEL_POINTS:           # n == 4 (cv2: P3P, out of scope) and n == 5: the kernel on all points
        return _solve(kernel, pws, p2, True)[1], np.ones(n, bool), np.inf
    subsets = cv_rng_subsets(n)
    best, best_mask, niters, near = 0, None, MAX_ITERS, np.inf
    it = 0
    while it < niters:
        idx = _subset(kernel, subsets[it])
        R, t = _solve(kernel, pws[idx], p2[idx], True)
        err = reprojection_errors(R, t, pws, p2)
        fin = np.isfinite(err)
        if fin.any():
            near = min(near, float(np.abs(err[fin].astype(np.float64) - float(THRESH2)).min()))
        mask = err <= THRESH2
        good = int(mask.sum())
        if good > max(best, MODEL_POINTS - 1):
            best, best_mask = good, mask
            niters = ransac_update_num_iters(CONFIDENCE, (n - good) / n, MODEL_POINTS, niters)
        it += 1
    if best_mask is None:
        return None, np.zeros(n, bool), near
    return _solve(kernel, pws[best_mask], p2[best_mask], False)[1], best_mask, near


def cam_trans_epnp(joints, cam, kernel="epnp"):
    """[n,71,3] joints, [n,3] cam -> (cam_trans [n,3] float32, inlier bitmask [n] int64 over the valid joints in order,
    near [n] float64 = the closest a joint came to the 400 px² threshold in any evaluated hypothesis)."""
    j3, p2, valid = pj2d_valid(joints, cam)
    n = len(j3)
    out, bits, near = np.zeros((n, 3), np.float32), np.zeros(n, np.int64), np.full(n, np.inf)
    for i in range(n):
        t, mask, near[i] = ransac_one(j3[i][valid[i]], p2[i][valid[i]], kernel)
        out[i] = INVALID if t is None else t.astype(np.float32)
        bits[i] = int(sum(1 << k for k in np.flatnonzero(mask)))
    return out, bits, near
