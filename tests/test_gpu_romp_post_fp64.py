"""ROMP's stages between the network and SMPL and after SMPL, each run through the C ABI on crafted device inputs and
compared with a plain float64 restatement of the same operation written here:
  b200romp_parse             bit-exact against a numpy restatement (5x5 max with -inf padding, value > thresh, score
                             descending / index ascending, 64 per frame, capacity cut) at its size and value edges
  rot6d_to_aa (via parse)    as ROTATIONS: Rodrigues_fp64(aa_gpu) against the fp64 Gram-Schmidt matrix, by geodesic angle
  b200romp_project(_frames)  pj2d_org, verts_camed_org, weak cam_trans against fp64, per-element bounds
  cam_trans least squares    against the fp64 normal equations on the kernel's own fp32 pixels (tight) and on fp64 pixels
                             (first-order perturbation bound)
  b200romp_one_euro_smooth   against the reference's outputs in both recurrences (--show_largest and tracked), and
                             against a float64 filter stepped from its own state over 300 frames x 256 slots
Bounds are per element, |err| <= g * 2^-24 * cond + tiny, cond the restatement on absolute values.  Every output buffer
is pre-filled with a sentinel and the rows past the count must keep it bit for bit.  Each check prints its worst
err / bound; each negative control mutates the restatement and must be rejected by the check it targets.  The tests
without the gpu marker run the fp32 CPU oracles through the same checks: the bounds admit a correct fp32 implementation
and reject the mutants on a machine without a GPU.

NaN cells: the reference's MaxPool2d propagates a NaN to all 25 cells around it, and its det * mask turns every
non-finite non-maximum into NaN, which torch.topk then ranks first, so a frame with non-finite cells loses its 64 slots
to garbage.  The kernel's rule is the one restated here: fmax ignores NaN neighbours, a NaN cell is never a peak, +inf
is an ordinary largest score, -inf never passes the threshold.

Worst err / bound seen on an H100 80 GB HBM3 at 700 W (fp32 CPU oracle in brackets): rot6d geodesic 0.59 (0.59), 0.09
on the near-parallel columns whose bound is the worst case of the Gram-Schmidt cancellation; pj2d_org / verts_camed_org
0.59 (0.66), weak cam_trans 0.25 (0.24); least squares on the kernel's pixels 0.93 (0.96), on fp64 pixels 0.11 (0.11: a
first-order worst case over 48 pixel roundings); One-Euro over 300 frames x 256 slots pose 0.51, betas 0.53, cam 0.43,
rotation 0.19 (0.48, 0.43, 0.38, 0.09 over 40 frames x 8 slots).  The GPU tests of this file take about 10 s after
start-up and peak at 151 MiB of device memory."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from oracle import romp_oracle as O
from oracle import temporal_oracle as TO
from romp_b200 import _lib

gpu = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
P = lambda t: C.c_void_p(t.data_ptr())
U = 2.0 ** -24
TINY = 1e-30
SENT = -7
F32, F64 = np.float32, np.float64
G_ROT = 16.0       # geodesic angle of rot6d_to_aa, times the amplification of the Gram-Schmidt step
G_PROJ = 4.0       # projection and weak cam_trans
G_PX = 1.5         # three roundings of half an ulp in (q*s + t + 1) * 256 entering the least squares
G_OE = 4.0         # per rounding step of the One-Euro recurrence
G_OE_ROT = 2.0     # filtered matrix -> axis-angle, as a rotation
BX_ROD = 4 * U     # fp32 axis-angle -> matrix (quaternion form), absolute per entry


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


# ====================================================================================================== 1. parse
def parse_ref(cm, pm, thresh, cap, n_betas, mutate=None):
    """numpy restatement of the parse; cm [B,1,S,S], pm [B,135+n_betas,S,S] -> dict of the rows."""
    B, S = cm.shape[0], cm.shape[-1]
    c = cm.reshape(B, S, S)
    pad = np.full((B, S + 4, S + 4), -np.inf, F32)
    pad[:, 2:-2, 2:-2] = c
    m = np.full_like(c, -np.inf)
    for dy in range(5):
        for dx in range(5):
            if mutate == "drop_cell" and (dy, dx) == (1, 3):
                continue
            m = np.fmax(m, pad[:, dy:dy + S, dx:dx + S])
    with np.errstate(invalid="ignore"):
        keep = (m == c) & ((c >= F32(thresh)) if mutate == "ge" else (c > F32(thresh)))
    bi, fi = [], []
    for b in range(B):
        idx = np.flatnonzero(keep[b])
        sc = c[b].ravel()[idx].astype(F64)
        order = np.lexsort((-idx if mutate == "ties_desc" else idx, -sc))
        idx = idx[order][:64]
        bi += [b] * len(idx); fi += idx.tolist()
    bi, fi = np.array(bi[:cap], np.int64), np.array(fi[:cap], np.int64)
    pp = pm.reshape(B, pm.shape[1], S * S)[bi, :, fi].reshape(len(bi), pm.shape[1])
    return dict(bi=bi, fi=fi, conf=c.reshape(B, -1)[bi, fi], pp=pp, cam=pp[:, :3], be=pp[:, 135:135 + n_betas],
                cp=np.stack([fi % S * 512 // S, fi // S * 512 // S], 1).astype(np.int64))


def parse_bufs(cap, n_betas):
    z = lambda *s, dt=torch.float32: torch.full(s, SENT, dtype=dt, device="cuda")
    return dict(count=z(1, dt=torch.int32), bi=z(cap, dt=torch.int64), fi=z(cap, dt=torch.int64), conf=z(cap),
                pp=z(cap, 135 + n_betas), cam=z(cap, 3), th=z(cap, 72), be=z(cap, n_betas), cp=z(cap, 2, dt=torch.int64))


def run_parse(cm, pm, thresh, cap, n_betas, bufs=None):
    """-> (count, every buffer in full on the host)."""
    lib, B, S = _lib.load(), cm.shape[0], cm.shape[-1]
    o = bufs or parse_bufs(cap, n_betas)
    c, p = dev(cm), dev(pm)
    ws = torch.zeros(int(lib.b200romp_parse_workspace_bytes(B)), dtype=torch.uint8, device="cuda")
    _lib.check(lib.b200romp_parse(P(c), P(p), B, S, n_betas, thresh, cap, P(o["count"]), P(o["bi"]), P(o["fi"]), P(o["conf"]),
                                  P(o["pp"]), P(o["cam"]), P(o["th"]), P(o["be"]), P(o["cp"]), P(ws), stream()), "parse")
    torch.cuda.synchronize()
    return int(o["count"].item()), {k: v.cpu().numpy() for k, v in o.items() if k != "count"}


def parse_diff(n, got, ref):
    """first difference between the kernel's rows [0,n) and the restatement, bits compared; None when identical."""
    if n != len(ref["bi"]):
        return f"count {n} != {len(ref['bi'])}"
    for k, r in ref.items():
        if got[k][:n].tobytes() != np.ascontiguousarray(r).astype(got[k].dtype).tobytes():
            return k
    return None


def tail_is_sentinel(n, got):
    return all((v[n:] == SENT).all() for v in got.values())


def parse_case(name, cm, pm, thresh, cap, n_betas, controls=()):
    n, got = run_parse(cm, pm, thresh, cap, n_betas)
    ref = parse_ref(cm, pm, thresh, cap, n_betas)
    d = parse_diff(n, got, ref)
    assert d is None, f"{name}: {d}"
    assert tail_is_sentinel(n, got), f"{name}: a row past the count was written"
    assert got["th"][:n, 66:].tobytes() == np.zeros((n, 6), F32).tobytes()            # +0.0 bits
    for mut in controls:
        assert parse_diff(n, got, parse_ref(cm, pm, thresh, cap, n_betas, mut)) is not None, f"{name}: control {mut} not rejected"
    print(f"{name}: {n} rows bit-exact, {cap - n} rows past the count untouched, controls rejected: {list(controls)}")
    return n, got


def dense_maps(B, S, n_betas, seed):
    rs = np.random.RandomState(seed)
    cm = rs.normal(0, 0.3, (B, 1, S, S)).astype(F32)
    pm = rs.normal(0, 1, (B, 135 + n_betas, S, S)).astype(F32)
    return cm, pm


def edge_maps():
    """-> (cm [6,1,64,64], thresh 0.25): non-finite cells, the threshold itself, corners, borders, 65 equal maxima."""
    cm = np.full((6, 1, 64, 64), -1.0, F32)
    f = cm[0, 0]
    f[10, 10] = np.inf; f[10, 12] = 0.9                      # +inf wins its window, 0.9 beside it is suppressed
    f[30, 30] = -np.inf; f[30, 33] = 0.5
    f[50, 50] = np.nan; f[50, 52] = 0.9; f[49, 49] = 0.3     # a NaN cell is no peak and hides nothing
    f = cm[1, 0]
    f[5, 5] = 0.25; f[20, 20] = np.nextafter(F32(0.25), F32(1)); f[40, 40] = np.nextafter(F32(0.25), F32(0))
    f = cm[2, 0]
    for k, (y, x) in enumerate([(0, 0), (0, 63), (63, 0), (63, 63), (0, 31), (63, 32), (31, 0), (32, 63)]):
        f[y, x] = 0.9 - 0.05 * k
    f[1, 1] = 0.95                                           # a larger neighbour suppresses the corner (0,0)
    f = cm[3, 0]
    f.reshape(-1)[np.arange(65) * 63] = 0.7                  # 65 equal maxima: the first 64 by index stay
    cm[4, 0] = 0.6                                           # plateau: every cell is a maximum
    cm[5, 0, 7, 7] = 0.7; cm[5, 0, 7, 8] = 0.7; cm[5, 0, 9, 9] = 0.7   # ties in one window, all kept, index ascending
    return cm


def zero_maps():
    """thresh 0: -0.0 beside +0.0 (neither is > 0), denormal peaks, a negative floor."""
    cm = np.zeros((2, 1, 64, 64), F32)
    cm[0, 0, 3, 3] = -0.0; cm[0, 0, 20, 20] = 1e-40; cm[0, 0, 40, 40] = 1.4e-45; cm[0, 0, 40, 42] = 2.8e-45
    cm[1] = -1e-40; cm[1, 0, 9, 9] = 0.0; cm[1, 0, 30, 30] = 1e-39
    return cm


def parse_controls_cpu():
    """every mutant changes the restatement's result on the inputs the GPU test uses."""
    cm, pm = dense_maps(3, 64, 10, 1)
    base = parse_ref(cm, pm, 0.25, 192, 10)
    assert not np.array_equal(base["fi"], parse_ref(cm, pm, 0.25, 192, 10, "drop_cell")["fi"])
    e = edge_maps()
    pe = dense_maps(6, 64, 10, 2)[1]
    base = parse_ref(e, pe, 0.25, 384, 10)
    assert len(parse_ref(e, pe, 0.25, 384, 10, "ge")["fi"]) == len(base["fi"]) + 1
    assert not np.array_equal(base["fi"], parse_ref(e, pe, 0.25, 384, 10, "ties_desc")["fi"])
    return base


def test_parse_restatement_cpu():
    """the restatement against the torch oracle where both are defined (finite maps), and its known answers."""
    cm, pm = dense_maps(3, 64, 10, 1)
    ref, o = parse_ref(cm, pm, 0.25, 192, 10), O.parsing_outputs(cm, pm, 0.25)
    assert np.array_equal(ref["bi"], o["pred_batch_ids"].numpy()) and np.array_equal(ref["fi"], o["flat_inds"].numpy())
    assert np.array_equal(ref["cp"], o["center_preds"].numpy()) and np.array_equal(ref["pp"], o["params_pred"].numpy())
    base = parse_controls_cpu()
    fi = lambda b: base["fi"][base["bi"] == b].tolist()
    assert fi(0) == [10 * 64 + 10, 50 * 64 + 52, 30 * 64 + 33, 49 * 64 + 49]
    assert fi(1) == [20 * 64 + 20]                                                  # bit-equal to thresh is not above it
    assert fi(2) == [65, 63, 63 * 64, 63 * 64 + 63, 31, 63 * 64 + 32, 31 * 64, 32 * 64 + 63]
    assert fi(3) == (np.arange(64) * 63).tolist() and fi(4) == list(range(64)) and fi(5) == [455, 456, 585]
    z = parse_ref(zero_maps(), dense_maps(2, 64, 10, 3)[1], 0.0, 128, 10)
    assert z["fi"].tolist() == [20 * 64 + 20, 40 * 64 + 42, 30 * 64 + 30]


@gpu
def test_parse_bit_exact_at_size_edges():
    cm, pm = dense_maps(64, 64, 10, 1)
    n, _ = parse_case("parse 64 frames x 64", cm, pm, 0.25, 4096, 10, ("drop_cell",))
    assert n == 4096                                                                # the benchmarked batch at capacity
    n, got = parse_case("parse capacity 4000", cm, pm, 0.25, 4000, 10)
    assert n == 4000 and got["bi"][-1] == 62                                        # the cut falls inside frame 62
    parse_case("parse batch 1", cm[:1], pm[:1], 0.25, 64, 10)
    for S, nb in ((64, 1), (32, 11), (5, 32), (1, 1), (32, 10), (5, 11)):
        c, p = dense_maps(3, S, nb, 10 + S + nb)
        n, _ = parse_case(f"parse map_size {S} n_betas {nb}", c, p, 0.1, 192, nb)
        assert n > 0
    c, p = dense_maps(300, 5, 1, 4)                                                 # the prefix sum strides by 256 frames
    n, got = parse_case("parse batch 300", c, p, 0.1, 300 * 64, 1)
    assert got["bi"][:n].max() == 299 and n > 300


@gpu
def test_parse_bit_exact_at_value_edges():
    parse_controls_cpu()
    e, pe = edge_maps(), dense_maps(6, 64, 10, 2)[1]
    parse_case("parse value edges", e, pe, 0.25, 384, 10, ("ge", "ties_desc"))
    parse_case("parse thresh 0, signed zeros and denormals", zero_maps(), dense_maps(2, 64, 10, 3)[1], 0.0, 128, 10)


@gpu
def test_parse_second_call_leaves_the_tail():
    cm, pm = dense_maps(2, 64, 10, 5)
    bufs = parse_bufs(160, 10)
    n1, first = run_parse(cm, pm, 0.25, 160, 10, bufs)
    assert n1 == 128
    cm2 = np.full((1, 1, 64, 64), -1.0, F32)
    cm2[0, 0, 3, 3] = 0.9; cm2[0, 0, 33, 40] = 0.8; cm2[0, 0, 60, 1] = 0.7
    n2, second = run_parse(cm2, pm[:1], 0.25, 160, 10, bufs)
    assert n2 == 3 and parse_diff(3, second, parse_ref(cm2, pm[:1], 0.25, 160, 10)) is None
    for k in first:
        assert second[k][3:].tobytes() == first[k][3:].tobytes(), k                 # rows 3..127 of the first call, then sentinel


# ====================================================================================================== 2. 6-D -> axis-angle
def rod64(aa):
    """exact Rodrigues, [N,3] -> [N,3,3] float64."""
    aa = np.asarray(aa, F64)
    th = np.linalg.norm(aa, axis=1)
    K = np.zeros((len(aa), 3, 3))
    with np.errstate(invalid="ignore"):                      # a non-finite aa stays non-finite and fails its check
        k = aa / np.maximum(th, 1e-300)[:, None]
        K[:, 0, 1], K[:, 0, 2], K[:, 1, 0], K[:, 1, 2], K[:, 2, 0], K[:, 2, 1] = -k[:, 2], k[:, 1], k[:, 2], -k[:, 0], -k[:, 1], k[:, 0]
        return np.eye(3) + np.sin(th)[:, None, None] * K + (1 - np.cos(th))[:, None, None] * (K @ K)


def gs64(x6, clamp=True):
    """fp64 rot6d_to_rotmat (utils.py:477-491) with F.normalize's eps clamp -> (R [N,3,3] columns b1 b2 b3, amplification)."""
    x = np.asarray(x6, F64).reshape(-1, 3, 2)
    a1, a2 = x[:, :, 0], x[:, :, 1]
    eps = 1e-6 if clamp else 0.0
    with np.errstate(all="ignore"):
        b1 = a1 / np.maximum(np.linalg.norm(a1, axis=1), eps)[:, None]
        u = a2 - (b1 * a2).sum(1, keepdims=True) * b1
        b2 = u / np.maximum(np.linalg.norm(u, axis=1), eps)[:, None]
        amp = np.linalg.norm(a1, axis=1) * np.linalg.norm(a2, axis=1) / np.linalg.norm(np.cross(a1, a2), axis=1)
    return np.stack([b1, b2, np.cross(b1, b2)], -1), np.maximum(1.0, amp)


def aa_from_rt64(Rt, mutate=None, nudge=(0.0, 0.0, 0.0)):
    """fp64 rotation_matrix_to_quaternion (utils.py:606-682) + quaternion_to_angle_axis (:554-604) on Rt [N,3,3] = R^T,
    NaN -> 0 (:551).  nudge moves the three branch comparisons (an fp32 matrix may sit on the other side of one).
    -> (aa [N,3], branch [N])."""
    m = lambda i, j: Rt[:, i, j]
    d2, d01, d0n1 = m(2, 2) + nudge[0] < 1e-6, m(0, 0) + nudge[1] > m(1, 1), m(0, 0) + nudge[2] < -m(1, 1)
    br = np.where(d2 & d01, 0, np.where(d2, 1, np.where(d0n1, 2, 3)))
    if mutate == "branch":
        br = np.where(br == 1, 2, br)
    t = [1 + m(0, 0) - m(1, 1) - m(2, 2), 1 - m(0, 0) + m(1, 1) - m(2, 2), 1 - m(0, 0) - m(1, 1) + m(2, 2), 1 + m(0, 0) + m(1, 1) + m(2, 2)]
    q = [np.stack([m(1, 2) - m(2, 1), t[0], m(0, 1) + m(1, 0), m(2, 0) + m(0, 2)], 1),
         np.stack([m(2, 0) - m(0, 2), m(0, 1) + m(1, 0), t[1], m(1, 2) + m(2, 1)], 1),
         np.stack([m(0, 1) - m(1, 0), m(2, 0) + m(0, 2), m(1, 2) + m(2, 1), t[2]], 1),
         np.stack([t[3], m(1, 2) - m(2, 1), m(2, 0) - m(0, 2), m(0, 1) - m(1, 0)], 1)]
    rows = np.arange(len(Rt))
    with np.errstate(all="ignore"):
        qq = np.stack(q, 0)[br, rows] / np.sqrt(np.stack(t, 0)[br, rows])[:, None] * 0.5
        s2 = (qq[:, 1:] ** 2).sum(1)
        s = np.sqrt(s2)
        two = 2 * np.where(qq[:, 0] < 0, np.arctan2(-s, -qq[:, 0]), np.arctan2(s, qq[:, 0]))
        aa = qq[:, 1:] * np.where(s2 > 0, two / s, 2.0)[:, None]
    return np.where(np.isnan(aa), 0.0, aa), br


def geodesic(Ra, Rb):
    return 2 * np.arcsin(np.minimum(1.0, np.linalg.norm(Ra - Rb, axis=(1, 2)) / (2 * np.sqrt(2))))


def axis_angle_matrix(axis, angle):
    return rod64(np.asarray(axis, F64)[None] / np.linalg.norm(axis) * angle)[0]


def rot6d_inputs():
    """-> dict group -> x6 [N,6] float32 (row-major [3,2]: column 0 = x[0::2], column 1 = x[1::2])."""
    rs = np.random.RandomState(17)
    axes = [(1, 0, 0), (0, 1, 0), (0, 0, 1), (1, 1, 0), (1, 0, 1), (0, 1, 1), (1, 1, 1), (-1, 1, 0), (1, -1, 1)] + [tuple(a) for a in rs.normal(size=(6, 3))]
    angles = [0.0, 1e-7, 1e-4, 1e-2, 0.5, 1.0, np.pi / 2, 2.0, 3.0, np.pi - 1e-2, np.pi - 1e-4, np.pi - 1e-6, np.pi]
    Rs = [axis_angle_matrix(a, sgn * th) for a in axes for th in angles for sgn in (1, -1)]
    Rs += [axis_angle_matrix((1, 0, 0), np.arccos(1e-6 + k * 2.5e-7)) for k in range(-3, 4)]       # m22 around the 1e-6 switch
    Rs += [axis_angle_matrix((0, 1, 0), np.arccos(1e-6 + k * 2.5e-7)) for k in range(-3, 4)]
    Rs = np.stack(Rs)
    six = lambda R, s1, s2: np.stack([R[:, :, 0] * s1, R[:, :, 1] * s2], -1).reshape(-1, 6)
    g = {"scaled": np.concatenate([six(Rs, s1, s2) for s1, s2 in ((1, 1), (1e-4, 1e-4), (1e4, 1e4), (1e-4, 1e4), (3, 0.2))])}
    sk = []
    for R in Rs[rs.choice(len(Rs), 40, replace=False)]:
        for e in (1e-1, 1e-2, 1e-3, 1e-4):
            sk.append(np.stack([R[:, 0], R[:, 0] * np.cos(e) + R[:, 1] * np.sin(e)], -1).reshape(6))
    g["skewed"] = np.stack(sk)
    g["clamped"] = np.concatenate([six(Rs, 1e-7, 1e-7), six(Rs, 1e-7, 1.0), six(Rs, 1.0, 1e-7)])    # below F.normalize's eps
    g["random"] = rs.normal(size=(4224 - len(g["scaled"]) - len(g["skewed"]) - len(g["clamped"]) - 8, 6))
    a = np.array([0.3, -0.5, 0.8])
    z = np.zeros(3)
    g["degenerate"] = np.stack([np.stack(c, -1).reshape(6) for c in
                                ((a, 2 * a), (a, -a), (z, a), (a, z), (z, z), (z, np.array([1.0, 0, 0])), (np.array([0, 1.0, 0]), z), (a, a))])
    return {k: v.astype(F32) for k, v in g.items()}


def assert_branches_populated(x6):
    R, _ = gs64(x6)
    Rt = R.transpose(0, 2, 1)
    _, br = aa_from_rt64(Rt)
    assert set(br.tolist()) == {0, 1, 2, 3}
    m00, m11, m22 = Rt[:, 0, 0], Rt[:, 1, 1], Rt[:, 2, 2]
    near = np.abs(m22 - 1e-6) < 1e-6
    assert (near & (m22 < 1e-6)).any() and (near & (m22 >= 1e-6)).any()
    assert ((np.abs(m00 - m11) < 1e-6) & (m22 < 1e-6)).any() and ((np.abs(m00 + m11) < 1e-6) & (m22 >= 1e-6)).any()


def check_rot6d(name, x6, aa, check=accepted, **mut):
    """aa [N,3] (an fp32 implementation's result for x6 [N,6] float32): the rotation it encodes against the fp64
    Gram-Schmidt matrix, and aa itself against the fp64 quaternion code below pi - 1e-2.  A column shorter than
    F.normalize's eps is divided by the eps, so that matrix is no rotation: the reference is then what the quaternion
    code makes of it, which is why both sides go through Rodrigues rather than the matrix itself."""
    R, amp = gs64(x6, clamp=not mut.get("no_clamp"))
    bound = G_ROT * U * amp
    if mut.get("against_matrix"):
        return check(f"{name} rotation (geodesic)", geodesic(rod64(aa), R), bound)
    # a branch comparison within 1e-6 of equality may fall either way in fp32: the branches agree on a rotation, but not
    # on the clamped matrices, so the nearest of the candidates counts
    e_rot, e_aa = np.full(len(aa), np.inf), np.full(len(aa), np.inf)
    for nudge in [(0, 0, 0)] + [tuple(sg * 1e-6 * (k == i) for k in range(3)) for i in range(3) for sg in (1, -1)]:
        ref, _ = aa_from_rt64(R.transpose(0, 2, 1), "branch" if mut.get("branch") else None, nudge)
        e_rot = np.fmin(e_rot, geodesic(rod64(aa), rod64(ref)))
        e_aa = np.fmin(e_aa, np.where(np.linalg.norm(ref, axis=1) < np.pi - 1e-2, np.abs(aa - ref).max(1), 0.0))
    r = check(f"{name} rotation (geodesic)", e_rot, bound)
    check(f"{name} axis-angle below pi - 1e-2", e_aa, 2 * bound)      # |d log| <= (angle / 2) / sin(angle / 2) < 1.6 there
    return r


def rot6d_checks(run):
    """run(x6 [N,6]) -> aa [N,3] float32."""
    g = rot6d_inputs()
    assert_branches_populated(np.concatenate([g["scaled"], g["skewed"]]))
    out = {k: run(v) for k, v in g.items()}
    for k in ("scaled", "skewed", "random"):
        check_rot6d(f"rot6d {k}", g[k], out[k])
        check_rot6d(f"rot6d {k} against the Gram-Schmidt matrix itself", g[k], out[k], against_matrix=True)
    check_rot6d("rot6d clamped", g["clamped"], out["clamped"])
    rejected("branch 2 where branch 1 applies", *_err_bound(check_rot6d, g["scaled"], out["scaled"], branch=True))
    rejected("normalize clamp left out", *_err_bound(check_rot6d, g["clamped"], out["clamped"], no_clamp=True))
    d = out["degenerate"]
    assert np.isfinite(d).all()                                                      # NaN -> 0, utils.py:551
    ex = O.rot6d_to_aa(torch.from_numpy(g["degenerate"])).numpy()                    # the fp32 oracle on the zero columns:
    assert np.array_equal(d[4:7], ex[4:7]), (d[4:7], ex[4:7])                        # zeros and unit axes involve no rounding,
    assert np.abs(d[2:4] - ex[2:4]).max() <= 4 * U * np.abs(ex[2:4]).max()           # normalising the other column does


def _err_bound(fn, x6, aa, **mut):
    got = []
    fn("", x6, aa, check=lambda n, e, b: got.append((e, b)) or 0.0, **mut)
    return got[0]


def test_rot6d_bounds_cpu():
    rot6d_checks(lambda x6: O.rot6d_to_aa(torch.from_numpy(x6)).numpy())
    x6 = rot6d_inputs()["scaled"]
    mine, _ = aa_from_rt64(gs64(x6)[0].transpose(0, 2, 1))                           # the restatement against the oracle in fp64
    theirs = O.rot6d_to_aa(torch.from_numpy(x6).double()).numpy()
    lo = np.linalg.norm(mine, axis=1) < np.pi - 1e-2
    assert np.abs(mine[lo] - theirs[lo]).max() < 1e-9


def rot6d_through_parse(x6):
    """plant 64 persons x 22 joints per frame, as many frames as x6 needs; -> aa [N,3] in x6's order."""
    n = len(x6)
    per = 64 * 22
    B = -(-n // per)
    x = np.zeros((B * per, 6), F32)
    x[:n] = x6
    x[n:, 0] = x[n:, 3] = 1.0
    cm = np.zeros((B, 1, 64, 64), F32)
    pm = np.zeros((B, 145, 64, 64), F32)
    for i in range(64):
        yy, xx = (i // 8) * 8, (i % 8) * 8
        cm[:, 0, yy, xx] = 0.99 - 0.01 * i
        pm[:, 3:135, yy, xx] = x.reshape(B, 64, 132)[:, i]
    cnt, got = run_parse(cm, pm, 0.25, B * 64, 10)
    assert cnt == B * 64 and (got["th"][:, 66:].view(np.int32) == 0).all()
    assert got["pp"][:, 3:135].tobytes() == x.reshape(B * 64, 132).tobytes()
    return got["th"][:, :66].reshape(-1, 3)[:n]


@gpu
def test_rot6d_to_axis_angle_as_rotations():
    rot6d_checks(rot6d_through_parse)


# ====================================================================================================== 3. projection
def pad_row(h, w):
    """padding_image's [top, bottom, left, right, h, w] for an h x w original."""
    size = max(h, w)
    top, left = (size - h) // 2, (size - w) // 2
    return np.array([top, size - h - top, left, size - w - left, h, w], F32)


PADS = [pad_row(512, 512), pad_row(1080, 1920), pad_row(2160, 3840), pad_row(1280, 720), pad_row(1, 1)]


def proj64(pts, cam, pad, mutate=None):
    """fp64 batch_orth_proj (utils.py:309-315) + convert_proejection_from_input_to_orgimg (post_parser.py:81-88);
    pts [n,k,3], cam [n,3], pad [6] or [n,6] -> (xy, z, bound_xy, bound_z)."""
    pts, cam, pad = np.asarray(pts, F64), np.asarray(cam, F64)[:, None], np.broadcast_to(np.asarray(pad, F64), (len(pts), 6))[:, None]
    top, left = pad[..., 0:1], pad[..., 2:3]
    size = (np.minimum if mutate == "min_size" else np.maximum)(pad[..., 4:5], pad[..., 5:6])
    if mutate == "swap":
        top, left = left, top
    off = np.concatenate([left, top], -1)
    xy = (pts[..., :2] * cam[..., :1] + cam[..., 1:] + 1) * size / 2 - off
    cond = (np.abs(pts[..., :2] * cam[..., :1]) + np.abs(cam[..., 1:]) + 1) * size / 2 + np.abs(off)
    return xy, (pts[..., 2] + 1) * size[..., 0] / 2, G_PROJ * U * cond, G_PROJ * U * (np.abs(pts[..., 2]) + 1) * size[..., 0] / 2


def weak64(cam):
    cam = np.asarray(cam, F64)
    with np.errstate(all="ignore"):
        w = np.stack([cam[:, 1] / cam[:, 0], cam[:, 2] / cam[:, 0], 1 / cam[:, 0]], 1) * 2
    return w


def people(n, seed, scales=(1e-3, 1.0, 30.0, -0.7)):
    """SMPL-like joints [n,71,3], a few vertices' worth of points, cams with the listed scales first."""
    rs = np.random.RandomState(seed)
    joints = (rs.uniform(-0.9, 0.9, (n, 71, 3)) * np.array([0.5, 1.0, 0.25])).astype(F32)
    cam = np.stack([rs.uniform(0.035, 1.8, n), rs.uniform(-0.8, 0.8, n), rs.uniform(-0.8, 0.8, n)], 1).astype(F32)
    cam[:min(n, len(scales)), 0] = scales[:n]
    return joints, cam


def check_projection(name, joints, cam, pad, pj, vco=None, verts=None, weak=None, check=accepted, mutate=None):
    xy, _, bxy, _ = proj64(joints, cam, pad, mutate)
    r = check(f"{name} pj2d_org", np.abs(pj - xy), bxy)
    if vco is not None:
        xy, z, bxy, bz = proj64(verts, cam, pad, mutate)
        check(f"{name} verts_camed_org xy", np.abs(vco[..., :2] - xy), bxy)
        check(f"{name} verts_camed_org z", np.abs(vco[..., 2] - z), bz)
    if weak is not None:
        w = weak64(cam)
        check(f"{name} weak cam_trans", np.abs(weak - w), G_PROJ * U * np.abs(w))
    return r


def run_project(joints, cam, pad, verts=None, d_count=None, want=("pj", "vco", "weak", "lsq"), batch_ids=None, pad_table=None):
    """b200romp_project (pad [6]) or, with batch_ids and pad_table, b200romp_project_frames -> full buffers on the host."""
    lib, n = _lib.load(), len(joints)
    j, c = dev(joints), dev(cam)
    v = dev(verts) if verts is not None else None
    z = lambda *s: torch.full(s, float(SENT), device="cuda")
    o = {"pj": z(n, 71, 2), "vco": z(n, verts.shape[1], 3) if verts is not None else None, "weak": z(n, 3), "lsq": z(n, 3)}
    o = {k: (t if k in want else None) for k, t in o.items()}
    p = lambda t: P(t) if t is not None else None
    cnt = None if d_count is None else torch.tensor([d_count], dtype=torch.int32, device="cuda")
    if batch_ids is None:
        rc = lib.b200romp_project(P(j), p(v), P(c), n, p(cnt), (C.c_float * 6)(*[float(x) for x in pad]), p(o["pj"]), p(o["vco"]),
                                  p(o["weak"]), p(o["lsq"]), stream())
    else:
        bi, pt = dev(batch_ids.astype(np.int64)), dev(pad_table)
        rc = lib.b200romp_project_frames(P(j), p(v), P(c), n, p(cnt), P(bi), P(pt), p(o["pj"]), p(o["vco"]), p(o["weak"]), p(o["lsq"]), stream())
    _lib.check(rc, "project")
    torch.cuda.synchronize()
    return {k: t.cpu().numpy() for k, t in o.items() if t is not None}


def test_projection_bounds_cpu():
    joints, cam = people(64, 3)
    for pad in PADS:
        o = O.project_outputs(torch.from_numpy(joints), torch.from_numpy(joints), cam, pad)
        check_projection(f"oracle fp32 {int(pad[4])}x{int(pad[5])}", joints, cam, pad, o["pj2d_org"].numpy(), o["verts_camed_org"].numpy(), joints,
                         O.cam_to_trans(cam).numpy())
    o = O.project_outputs(torch.from_numpy(joints), None, cam, PADS[1])
    for mut in ("min_size", "swap"):
        check_projection(mut, joints, cam, PADS[1], o["pj2d_org"].numpy(), check=rejected, mutate=mut)


@gpu
def test_projection_against_fp64():
    rs = np.random.RandomState(8)
    for n, pad in ((1, PADS[0]), (5, PADS[1]), (5, PADS[2]), (37, PADS[3]), (5, PADS[4]), (4096, PADS[1])):
        joints, cam = people(n, n)
        verts = rs.uniform(-1, 1, (n, 6890, 3)).astype(F32) if n <= 37 else None
        o = run_project(joints, cam, pad, verts)
        check_projection(f"project n={n} {int(pad[4])}x{int(pad[5])}", joints, cam, pad, o["pj"], o.get("vco"), verts, o["weak"])
    joints, cam = people(64, 3)
    verts = rs.uniform(-1, 1, (64, 6890, 3)).astype(F32)
    full = run_project(joints, cam, PADS[1], verts)
    for mut in ("min_size", "swap"):
        check_projection(mut, joints, cam, PADS[1], full["pj"], check=rejected, mutate=mut)
    for d_count, rows in ((0, 0), (37, 37), (1000, 64)):                              # device count: below, and above n (clamped)
        o = run_project(joints, cam, PADS[1], verts, d_count=d_count)
        for k, v in o.items():
            assert v[:rows].tobytes() == full[k][:rows].tobytes() and (v[rows:] == SENT).all(), (d_count, k)
    for drop in ("pj", "vco", "weak", "lsq"):                                         # every optional output NULL in turn
        o = run_project(joints, cam, PADS[1], verts, want=[k for k in full if k != drop])
        assert set(o) == set(full) - {drop} and all(o[k].tobytes() == full[k].tobytes() for k in o), drop
    # s = 0: the reference divides by it too; the same non-finite pattern, kept out of every bound
    cam0 = cam.copy(); cam0[:3, 0] = 0.0; cam0[1, 1] = 0.0; cam0[2, 1:] = (-0.5, 0.0)
    o = run_project(joints, cam0, PADS[1])
    with np.errstate(all="ignore"):
        w32 = np.stack([cam0[:, 1] / cam0[:, 0], cam0[:, 2] / cam0[:, 0], F32(1) / cam0[:, 0]], 1) * F32(2)
    assert np.array_equal(np.isnan(o["weak"]), np.isnan(w32)) and np.array_equal(o["weak"][:3][np.isinf(w32[:3])], w32[:3][np.isinf(w32[:3])])
    assert np.isnan(w32[:3]).any() and np.isinf(w32[:3]).any() and np.isfinite(o["pj"]).all()


@gpu
def test_project_frames_equals_project_per_frame():
    rs = np.random.RandomState(9)
    table = np.stack([pad_row(int(h), int(w)) for h, w in zip(rs.randint(1, 4000, 64), rs.randint(1, 4000, 64))])
    table[:5] = PADS
    bi = np.sort(np.concatenate([np.repeat([0, 1, 2, 3, 4, 7, 7, 7, 20, 63], 6), rs.choice([9, 30, 31, 62], 40)]))   # frames skipped and repeated
    n = len(bi)
    joints, cam = people(n, 12)
    verts = rs.uniform(-1, 1, (n, 6890, 3)).astype(F32)
    o = run_project(joints, cam, None, verts, batch_ids=bi, pad_table=table)
    check_projection("project_frames", joints, cam, table[bi], o["pj"], o["vco"], verts, o["weak"])
    for f in np.unique(bi):
        r = bi == f
        one = run_project(joints[r], cam[r], table[f], verts[r])
        assert all(one[k].tobytes() == o[k][r].tobytes() for k in one), f
    part = run_project(joints, cam, None, verts, d_count=37, batch_ids=bi, pad_table=table)
    assert all(v[:37].tobytes() == o[k][:37].tobytes() and (v[37:] == SENT).all() for k, v in part.items())


# ====================================================================================================== 4. cam_trans least squares
def lsq_ref(joints, cam, px_mode, focal=F64(F32(443.4)), ignore_z=False):
    """estimate_translation_np (utils.py:347-389, unit weights) behind the validity mask of :404-421, normal equations
    and solve in fp64.  px_mode: how (q*s + t + 1) * 256 is formed - "f32" rounds every operation, "fma" rounds q*s + t
    once (the contraction a compiler may choose), "f64" keeps doubles.
    -> (x [n,3], first-order bound [n,3] for errors of G_PX roundings in the pixels, cond(A) [n], valid counts [n])."""
    q, c = joints[:, :24], cam[:, None]
    with np.errstate(all="ignore"):
        if px_mode == "f32":
            px = ((q[..., :2] * c[..., :1] + c[..., 1:]) + F32(1)) * F32(256)
        elif px_mode == "fma":
            px = ((q[..., :2].astype(F64) * c[..., :1].astype(F64) + c[..., 1:].astype(F64)).astype(F32) + F32(1)) * F32(256)
        else:
            px = (q[..., :2].astype(F64) * c[..., :1].astype(F64) + c[..., 1:].astype(F64) + 1) * 256
        valid = px[..., 1] > -2
    if not ignore_z:
        valid &= q[..., 2] != F32(-2)
    x, bound, cond = np.full((len(q), 3), -1.0), np.zeros((len(q), 3)), np.ones(len(q))
    Fo, Oc = float(focal), 256.0
    for i in np.flatnonzero(valid.sum(1) >= 4):
        v = valid[i]
        p, X = px[i][v].astype(F64), q[i][v].astype(F64)
        e = G_PX * U * (np.abs(X[:, :2] * F64(cam[i, 0])) + np.abs(F64(cam[i, 1:])) + 1) * 256
        A, b, dA, db = np.zeros((3, 3)), np.zeros(3), np.zeros((3, 3)), np.zeros(3)
        for k in range(2):
            Q = np.zeros((len(p), 3)); Q[:, k] = Fo; Q[:, 2] = Oc - p[:, k]
            cc = (p[:, k] - Oc) * X[:, 2] - Fo * X[:, k]
            A += Q.T @ Q; b += Q.T @ cc
            dA[k, 2] += Fo * e[:, k].sum(); dA[2, k] = dA[k, 2]
            dA[2, 2] += (2 * np.abs(Q[:, 2]) * e[:, k]).sum()
            db[k] += (Fo * np.abs(X[:, 2]) * e[:, k]).sum()
            db[2] += (e[:, k] * (np.abs(cc) + np.abs(Q[:, 2] * X[:, 2]))).sum()
        x[i] = np.linalg.solve(A, b)
        cond[i] = np.linalg.cond(A)
        bound[i] = np.abs(np.linalg.inv(A)) @ (db + dA @ np.abs(x[i])) + U * np.abs(x[i])
    return x, bound, cond, valid.sum(1)


def lsq_people():
    """-> joints [n,71,3], cam [n,3], and the rows of the named edge cases."""
    rs = np.random.RandomState(23)
    n = 256
    joints, cam = people(n, 23, scales=())
    depth = np.exp(rs.uniform(0, np.log(50), n))                                     # 1 m .. 50 m
    cam[:, 0] = (2 * 443.4 / 512 / depth).astype(F32)
    rows = {}
    joints[0, 4:24, 2] = -2; rows["4 valid"] = 0
    joints[1, 3:24, 2] = -2; rows["3 valid"] = 1
    joints[2, :21, 1] = (-1.05 - cam[2, 2]) / cam[2, 0]; rows["py <= -2"] = 2        # 3 valid -> -1
    joints[3, :20, 1] = np.nan; rows["py NaN"] = 3                                   # 4 valid
    joints[4, 5:12, 2] = -2; joints[4, 12:15, 1] = np.nan; rows["mixed"] = 4
    joints[5, :24, 2] = 0.3 + 1e-4 * rs.normal(size=24); rows["nearly planar"] = 5
    t = np.linspace(-0.8, 0.8, 24)
    joints[6, :24] = np.stack([0.4 * t, t, 0.1 * t], 1) + 1e-4 * rs.normal(size=(24, 3)); rows["nearly collinear"] = 6
    joints[7, :24] *= 1e-3; rows["all joints in one pixel"] = 7
    return joints, cam, rows


def check_lsq(name, joints, cam, got, check=accepted, focal_a=F64(F32(443.4)), **mut):
    """focal_a: the focal length of the implementation under test (the kernel holds 443.4 as a float)."""
    rows = np.arange(len(joints))
    xa = [lsq_ref(joints, cam, m, **{"focal": focal_a, **mut}) for m in ("f32", "fma")]
    inv = xa[0][3] < 4
    assert (got[inv].view(np.int32) == np.array(-1.0, F32).view(np.int32)).all() if not mut else True   # the three -1 values, bits
    # (a) the kernel's own pixels: fp64 solve rounded once to fp32; whichever contraction the compiler chose, per person
    ea = [np.abs(got - x) for x, _, _, _ in xa]
    ba = [U * np.abs(x) + 256 * 2.0 ** -53 * c[:, None] * np.abs(x).max(1, keepdims=True) for x, _, c, _ in xa]
    pick = np.argmin([(e / (b + TINY)).max(1) for e, b in zip(ea, ba)], 0)
    r = check(f"{name} (a) fp32 pixels, fp64 solve", np.stack(ea)[pick, rows], np.stack(ba)[pick, rows])
    if mut:
        return r
    print(f"    persons nearer the uncontracted pixels: {int((pick == 0).sum())}, the contracted: {int((pick == 1).sum())}")
    xb, bb, cond, _ = lsq_ref(joints, cam, "f64", focal=443.4)
    ok = ~inv
    check(f"{name} (b) fp64 pixels", np.abs(got[ok] - xb[ok]), bb[ok] + 4e-8 * np.abs(xb[ok]))       # + focal 443.4 as a float
    return r, cond


def lsq_checks(run, **kw):
    joints, cam, rows = lsq_people()
    got = run(joints, cam)
    _, cond = check_lsq("cam_trans lsq", joints, cam, got, **kw)
    valid = lsq_ref(joints, cam, "f32")[3]
    for k, i in rows.items():
        print(f"    {k}: {valid[i]} valid joints, cond(A) {cond[i]:.3e}, cam_trans {got[i]}")
    assert valid[rows["4 valid"]] == 4 and valid[rows["py NaN"]] == 4 and valid[rows["3 valid"]] == 3 and valid[rows["py <= -2"]] == 3
    assert (got[[1, 2]] == -1).all() and (got[[0, 3]] != -1).all()
    check_lsq("focal 443.0", joints, cam, got, check=rejected, focal=443.0)
    check_lsq("mask ignores z == -2", joints, cam, got, check=rejected, ignore_z=True, **kw)
    return joints, cam, got


def test_cam_trans_lsq_bounds_cpu():
    lsq_checks(lambda j, c: O.project_outputs(torch.from_numpy(j), None, c, PADS[0])["cam_trans"].numpy(), focal_a=443.4)


@gpu
def test_cam_trans_lsq_against_fp64():
    joints, cam, full = lsq_checks(lambda j, c: run_project(j, c, PADS[0], want=("lsq",))["lsq"])
    for d_count, rows in ((0, 0), (37, 37), (1000, 256)):
        o = run_project(joints, cam, PADS[0], d_count=d_count, want=("lsq",))["lsq"]
        assert o[:rows].tobytes() == full[:rows].tobytes() and (o[rows:] == SENT).all()


# ====================================================================================================== 5. One-Euro
NCH, K_POSE, K_BETA, K_CAM = 97, 9, 78, 94       # global-rotation matrix | body pose | betas (16) | cam


def oe_rod64(aa):
    """fp64 utils.batch_rodrigues (:493-505) + quat2mat (:507-533), [n,3] -> [n,9]."""
    aa = np.asarray(aa, F64)
    nrm = np.linalg.norm(aa + 1e-8, axis=1, keepdims=True)
    q = np.concatenate([np.cos(nrm / 2), np.sin(nrm / 2) * aa / nrm], 1)
    w, x, y, z = (q / np.linalg.norm(q, axis=1, keepdims=True)).T
    return np.stack([w * w + x * x - y * y - z * z, 2 * x * y - 2 * w * z, 2 * w * y + 2 * x * z, 2 * w * z + 2 * x * y,
                     w * w - x * x + y * y - z * z, 2 * y * z - 2 * w * x, 2 * x * z - 2 * w * y, 2 * w * x + 2 * y * z,
                     w * w - x * x - y * y + z * z], 1)


class OneEuro64:
    """fp64 OneEuroFilter (utils.py:217-246) for every slot and channel at once, stepped from its own state, with a
    running first-order bound on what an fp32 implementation of the same recurrence may differ by.  tracked: the pose,
    betas and cam filters keep their smoothed value as prev_raw (the reference's row views, romp/main.py:152-154)."""

    def __init__(self, slots, coeff, tracked, n_betas=10):
        self.raw, self.px, self.pdx = (np.zeros((slots, NCH)) for _ in range(3))
        self.b_raw, self.b_px, self.b_pdx = (np.zeros((slots, NCH)) for _ in range(3))
        self.seen = np.zeros(slots, bool)
        self.mincut = np.concatenate([np.full(K_BETA, float(coeff)), np.full(16, 0.6), np.full(3, 1.6)])
        self.aliased = np.arange(NCH) >= K_POSE if tracked else np.zeros(NCH, bool)
        self.n_betas = n_betas

    def pack(self, thetas, betas, cam):
        n = len(thetas)
        x, bx = np.zeros((n, NCH)), np.zeros((n, NCH))
        x[:, :K_POSE], bx[:, :K_POSE] = oe_rod64(thetas[:, :3]), BX_ROD
        x[:, K_POSE:K_BETA], x[:, K_BETA:K_BETA + self.n_betas], x[:, K_CAM:] = thetas[:, 3:], betas[:, :self.n_betas], cam
        return x, bx

    def step(self, slots, thetas, betas, cam):
        """-> (y [n,97], bound [n,97]) for the persons in slots (all distinct)."""
        x, bx = self.pack(thetas, betas, cam)
        k = 30.0 / (2 * np.pi)
        alpha = lambda c: 1.0 / (1.0 + k / c)
        s, raw, px, pdx = self.seen[slots][:, None], self.raw[slots], self.px[slots], self.pdx[slots]
        ad = alpha(1.0)
        dx = (x - raw) * 30
        b_dx = 30 * (bx + self.b_raw[slots]) + G_OE * U * 30 * (np.abs(x) + np.abs(raw))
        edx = ad * dx + (1 - ad) * pdx
        b_edx = ad * b_dx + (1 - ad) * self.b_pdx[slots] + G_OE * U * (np.abs(ad * dx) + np.abs((1 - ad) * pdx))
        cut = self.mincut + 0.7 * np.abs(edx)
        a = alpha(cut)
        b_a = 0.7 * b_edx * k / (cut + k) ** 2 + G_OE * U * a
        y = a * x + (1 - a) * px
        b_y = b_a * np.abs(x - px) + a * bx + (1 - a) * self.b_px[slots] + G_OE * U * (np.abs(a * x) + np.abs((1 - a) * px))
        y, b_y, edx, b_edx = np.where(s, y, x), np.where(s, b_y, bx), np.where(s, edx, 0.0), np.where(s, b_edx, 0.0)
        self.raw[slots], self.b_raw[slots] = np.where(self.aliased, y, x), np.where(self.aliased, b_y, bx)
        self.px[slots], self.b_px[slots], self.pdx[slots], self.b_pdx[slots] = y, b_y, edx, b_edx
        self.seen[slots] = True
        return y, b_y

    def reset(self, slot):
        self.seen[slot] = False


def check_one_euro(name, oe, y, b_y, thetas, betas, cam, worst, check=accepted):
    """thetas/betas/cam: an fp32 implementation's smoothed outputs for the step that gave (y, b_y); worst: dict of ratios."""
    ref_aa, _ = aa_from_rt64(y[:, :K_POSE].reshape(-1, 3, 3).transpose(0, 2, 1))     # the filtered matrix is not orthonormal
    groups = {"rotation": (geodesic(rod64(thetas[:, :3]), rod64(ref_aa)), G_OE_ROT * (np.linalg.norm(b_y[:, :K_POSE], axis=1) + 4 * U)),
              "pose": (np.abs(thetas[:, 3:] - y[:, K_POSE:K_BETA]), b_y[:, K_POSE:K_BETA]),
              "betas": (np.abs(betas[:, :oe.n_betas] - y[:, K_BETA:K_BETA + oe.n_betas]), b_y[:, K_BETA:K_BETA + oe.n_betas]),
              "cam": (np.abs(cam - y[:, K_CAM:]), b_y[:, K_CAM:])}
    for g, (e, b) in groups.items():
        r = float(np.max(e / (b + TINY))) if np.all(e <= b + TINY) else float("inf")
        worst[g] = max(worst.get(g, 0.0), r)


def walks(T, n, seed, n_betas=10):
    """random walks of n persons over T frames; every eighth person's global rotation passes through pi."""
    rs = np.random.RandomState(seed)
    th = (np.cumsum(rs.normal(0, 0.05, (T, n, 72)), 0) + rs.normal(0, 0.5, (1, n, 72))).astype(F32)
    ax = rs.normal(size=(n, 3)); ax /= np.linalg.norm(ax, axis=1, keepdims=True)
    w = np.arange(n) % 8 == 0
    th[:, w, :3] = (ax[None, w] * (np.linspace(2.6, 3.7, T)[:, None, None] + rs.normal(0, 0.01, (T, int(w.sum()), 1)))).astype(F32)
    be = np.cumsum(rs.normal(0, 0.03, (T, n, n_betas)), 0).astype(F32)
    ca = (np.array([0.8, 0.0, 0.1]) + np.cumsum(rs.normal(0, 0.01, (T, n, 3)), 0)).astype(F32)
    return th, be, ca


class Tracks:
    """b200romp_tracks handle + one call of b200romp_one_euro_smooth on host arrays."""

    def __init__(self, slots):
        self.lib = _lib.load()
        self.h = self.lib.b200romp_tracks_create(0, slots)
        assert self.h

    def reset(self, slot=-1):
        _lib.check(self.lib.b200romp_tracks_reset(self.h, slot, stream()), "tracks_reset")

    def smooth(self, slots, thetas, betas, cam, coeff, tracked, n_betas=10, d_count=None, n=None):
        """-> smoothed copies (thetas, betas, cam); betas [n, betas_stride]."""
        s, th, be, ca = dev(np.asarray(slots, np.int32)), dev(thetas), dev(betas), dev(cam)
        cnt = None if d_count is None else torch.tensor([d_count], dtype=torch.int32, device="cuda")
        _lib.check(self.lib.b200romp_one_euro_smooth(self.h, P(s), n or len(slots), P(cnt) if cnt is not None else None, P(th), P(be),
                                                     betas.shape[1], n_betas, P(ca), coeff, 30.0, int(tracked), stream()), "one_euro")
        torch.cuda.synchronize()
        return th.cpu().numpy(), be.cpu().numpy(), ca.cpu().numpy()

    def close(self):
        self.lib.b200romp_tracks_destroy(self.h)


def fixture_errors(z, smooth_rows):
    """per-frame max |err| of smooth_rows(ids [n], thetas, betas, cam) -> (thetas, betas, cam) over a golden fixture."""
    errs = []
    for t in range(len(z["thetas"])):
        n = int(z["n"][t]) if "n" in z else z["thetas"].shape[1]
        ids = z["ids"][t, :n] if "ids" in z else np.arange(1, n + 1)
        th, be, ca = smooth_rows(ids, z["thetas"][t, :n], z["betas"][t, :n], z["cam"][t, :n])
        errs.append(max(np.abs(th - z["out_thetas"][t, :n]).max(), np.abs(be - z["out_betas"][t, :n]).max(), np.abs(ca - z["out_cam"][t, :n]).max()))
    return np.array(errs)


def golden(name):
    z = np.load(os.path.join(HERE, "golden", name))
    return {k: z[k] for k in z.files}


@gpu
def test_one_euro_reference_recurrences():
    """the kernel against the reference's own outputs: --show_largest fixture with tracked = 0, tracked fixture with
    tracked = 1; each fixture rejects the other recurrence from every track's third sample on."""
    tr = Tracks(16)
    slot_of = np.array([-1, 5, 0, 9, 14, 2, 7], np.int32)                             # id -> arbitrary, non-contiguous slots
    for name, mode in (("one_euro.npz", 0), ("one_euro_tracked.npz", 1)):
        z = golden(name)
        for tracked in (mode, 1 - mode):
            tr.reset()
            err = fixture_errors(z, lambda ids, th, be, ca: tr.smooth(slot_of[ids], th, be, ca, 3.0, tracked))
            print(f"{name} tracked={tracked}: max |kernel - reference| per frame, first 5: {err[:5]}, overall {err.max():.2e}")
            if tracked == mode:
                assert err.max() < 3e-5
            else:
                assert err[:2].max() < 3e-5 and (err[2:] > 3e-5).all() and err[2] > 1e-3
    tr.close()


def one_euro_long_run(smooth, T, n_per, signals, coeff, tracked):
    """smooth(slots, thetas, betas, cam) -> smoothed, an fp32 implementation holding slots' state; stepped beside the fp64
    filter on the same inputs, rows in a new order every frame."""
    n = n_per * signals
    th, be, ca = walks(T, n, 31 + tracked)
    oe, worst, rs = OneEuro64(n, coeff, tracked), {}, np.random.RandomState(5)
    for t in range(T):
        order = rs.permutation(n)
        slots = order.astype(np.int32)
        y, b_y = oe.step(slots, th[t, order], be[t, order], ca[t, order])
        check_one_euro("", oe, y, b_y, *smooth(slots, th[t, order], be[t, order], ca[t, order]), worst)
    print(f"one-euro {T} frames x {n} slots, smooth_coeff {coeff}, tracked={tracked}: worst err/bound " +
          ", ".join(f"{k} {v:.3f}" for k, v in worst.items()))
    assert max(worst.values()) <= 1.0, worst
    return worst


class OracleFilters:
    """oracle/temporal_oracle.py (fp32) behind the same call as the kernel."""

    def __init__(self, coeff, tracked):
        self.f, self.coeff, self.tracked = {}, coeff, tracked

    def __call__(self, slots, th, be, ca):
        th, be, ca = th.copy(), be.copy(), ca.copy()
        for r, s in enumerate(slots.tolist()):
            f = self.f.setdefault(s, TO.make_filters(self.coeff))
            if self.tracked:
                TO.smooth_tracked(f, th[r], be[r], ca[r])
            else:
                th[r], be[r], ca[r] = TO.smooth(f, th[r].copy(), be[r].copy(), ca[r].copy())
        return th, be, ca


@pytest.mark.parametrize("tracked", [0, 1])
def test_one_euro_bounds_cpu(tracked):
    one_euro_long_run(OracleFilters(3.0, tracked), 40, 8, 1, 3.0, tracked)
    with pytest.raises(AssertionError):                                               # the other recurrence is rejected
        one_euro_long_run(OracleFilters(3.0, 1 - tracked), 40, 8, 1, 3.0, tracked)


@gpu
@pytest.mark.parametrize("tracked", [0, 1])
@pytest.mark.parametrize("coeff", [3.0, 0.5])
def test_one_euro_against_fp64_over_300_frames(tracked, coeff):
    tr = Tracks(256)
    one_euro_long_run(lambda s, th, be, ca: tr.smooth(s, th, be, ca, coeff, tracked), 300, 64, 4, coeff, tracked)
    tr.close()


@gpu
@pytest.mark.parametrize("tracked", [0, 1])
def test_one_euro_edges(tracked):
    """slot -1 and rows past the device count stay bit-identical; betas_stride > n_betas leaves the pad columns; a slot
    reset re-initialises that slot only; two launches on disjoint slots equal one."""
    T, n, nb = 12, 24, 11
    th, be11, ca = walks(T, n, 77, n_betas=nb)
    be16 = np.full((T, n, 16), float(SENT), F32); be16[..., :nb] = be11
    slots = (np.arange(n) * 3 % 64).astype(np.int32)
    slots[[4, 17]] = -1
    a, b, c, oe = Tracks(64), Tracks(64), Tracks(64), OneEuro64(64, 3.0, tracked, n_betas=nb)
    live = slots >= 0
    worst = {}
    for t in range(T):
        if t == 6:                                                                    # forget one slot in the middle
            for tr in (a, b, c):
                tr.reset(int(slots[2]))
            oe.reset(int(slots[2]))
        cnt = 20 if t % 2 else None                                                   # rows 20.. past the device count every other frame
        rows = live & (np.arange(n) < (cnt or n))
        o11 = a.smooth(slots, th[t], be11[t], ca[t], 3.0, tracked, n_betas=nb, d_count=cnt)
        o16 = b.smooth(slots, th[t], be16[t], ca[t], 3.0, tracked, n_betas=nb, d_count=cnt)
        lo, hi = slots.copy(), slots.copy()                                           # the same step as two launches, one stream
        lo[10:], hi[:10] = -1, -1
        h1 = c.smooth(lo, th[t], be16[t], ca[t], 3.0, tracked, n_betas=nb, d_count=cnt)
        h2 = c.smooth(hi, *h1, 3.0, tracked, n_betas=nb, d_count=cnt)
        for x, y in zip(o16, h2):
            assert x.tobytes() == y.tobytes()
        assert o16[0].tobytes() == o11[0].tobytes() and o16[2].tobytes() == o11[2].tobytes()
        assert o16[1][..., :nb].tobytes() == o11[1].tobytes() and (o16[1][..., nb:] == SENT).all()
        for got, src in zip(o11, (th[t], be11[t], ca[t])):
            assert got[~rows].tobytes() == src[~rows].tobytes()                       # untouched rows, bits
        if t == 6:                                                                    # the reset slot passes its input through
            assert o11[1][2].tobytes() == be11[t, 2].tobytes() and o11[2][2].tobytes() == ca[t, 2].tobytes()
            assert o11[0][2, 3:].tobytes() == th[t, 2, 3:].tobytes() and o11[2][3].tobytes() != ca[t, 3].tobytes()
        y, b_y = oe.step(slots[rows], th[t][rows], be11[t][rows], ca[t][rows])
        check_one_euro("", oe, y, b_y, o11[0][rows], o11[1][rows], o11[2][rows], worst)
    print(f"one-euro edges tracked={tracked}: worst err/bound " + ", ".join(f"{k} {v:.3f}" for k, v in worst.items()))
    assert max(worst.values()) <= 1.0, worst
    for tr in (a, b, c):
        tr.close()
