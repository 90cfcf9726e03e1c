"""The SMPL forward on the GPU, stage by stage, against a float64 run of the oracle (oracle/romp_oracle.smpl_forward).

Each stage is checked on the GPU's own inputs to that stage, so that each bound covers one kernel:
  - pose kernel: the features [betas | R[1:]-I], the relative transforms A[24][3x4] and joints 0-23 against float64 from the
    same betas and thetas.  Yardstick: the fp32 oracle's own distance from float64; the GPU may be POSE_FACTOR times as far,
    plus a floor of POSE_FLOOR.  The fp16 hi / lo split of the features (the blend GEMM's left operand) must be exact.
  - blend GEMM: v_posed = v_template + f B in float64 with the GPU's features f;
  - skinning GEMM: verts = (W A) [v_posed; 1] in float64 with the GPU's A and v_posed;
  - joints kernel: joints 24-44 are the picked vertices, bit for bit; joints 45-70 the regressors applied in float64 to the
    GPU's verts.  With root_align the root and the subtraction are compared bit for bit with the GPU's non-aligned run.
  - end to end: verts and joints against float64 SMPL from betas and thetas.
Both GEMMs run on the tensor cores with a 3-term fp16 split: x = hi + lo, x y ~ hi hi' + lo hi' + hi lo'.  Each GEMM stage gets
  1. a per-element bound that is never exceeded (split_gemm_bound): split representation 3 2^-22 S, fp32 accumulation
     U_TC (3K + 3) S, with S = sum |a||b|, an absolute allowance for fp16 subnormal hi / lo parts, plus output rounding.
     U_TC = 2^-23: round-to-nearest of the tensor cores' fp32 accumulation is not documented, so a full ulp per add.
     This catches indexing, masking and layout errors;
  2. a global maximum error per stage (LIMITS), set from the CPU emulation of the exact split with headroom, far below what
     a lost cross term or a flushed subnormal costs.  test_split_calibration_cpu shows that the emulation passes both
     checks and that the emulated mutations (a dropped cross term, hi only, lo flushed to zero where subnormal) fail them.
Every check prints its max error and max err/bound, so the margins are visible with -s.

The 65,536-person run holds 5.4 GB of verts and 5.6 GB of workspace; the float64 references run in chunks of CHUNK persons.
Measured on one H100 80GB HBM3 (400 W power limit): peak torch allocation 11.5 GiB in the 65,536-person test (8.3 s), the
whole GPU part of this file 22 s.
"""
import math
import time

import numpy as np
import pytest
import torch

from oracle import romp_oracle as O
from romp_b200 import synth

V, NJ, COLS = 6890, 24, 6890 * 3
DEV = "cuda"                   # where the GPU checks keep their tensors and run the float64 references
CHUNK = 256                    # persons per float64 reference chunk
SENTINEL = 123.0               # initial value of every output row: rows at or past the person count must keep it

# fp32 arithmetic
U32 = 2.0 ** -24               # CUDA-core fp32 (round to nearest)
U_TC = 2.0 ** -23              # tensor-core fp32 accumulation (rounding mode not documented: a full ulp per add)
SPLIT_REL = 3 * 2.0 ** -22     # x = hi + lo + d, |d| <= 2^-22 |x|; the dropped lo*lo' <= 2^-22 |x||y|
SUBNORMAL = 2.0 ** -24         # absolute error of an fp16 part in the subnormal range (half an ulp is 2^-25), per |operand|
POSE_FACTOR, POSE_FLOOR = 4.0, 4 * 2.0 ** -24

# Global max |err| per stage and pack.  The CPU emulation of the exact 3-term split leaves, on the edge inputs
# (test_split_calibration_cpu), v_posed / verts / end-to-end verts: synthetic 1.2e-6 / 2.2e-7 / 1.1e-6, real_scale
# 3.2e-6 / 6.3e-7 / 2.7e-6, wide_range 1.4e-6 / 5.8e-7 / 1.5e-6.  The kernels leave about twice that on v_posed (measured on
# one H100 80GB HBM3 at a 400 W power limit, over every shape of this file: synthetic 2.5e-6 / 5.7e-7 / 2.1e-6, real_scale
# 7.4e-6 / 1.2e-6 / 6.9e-6, wide_range 3.7e-6 / 8.8e-7 / 4.1e-6): the tensor cores' fp32 accumulation does not round to
# nearest.  The limits are about 3-4x the kernels' error, and a dropped cross term, hi only or a flushed subnormal lo costs at
# least 5.7e-5 on v_posed and 2.2e-4 on verts.
LIMITS = {
    "synthetic": dict(v_posed=8e-6, verts=2e-6, e2e=8e-6),
    "real_scale": dict(v_posed=2.5e-5, verts=4e-6, e2e=2.5e-5),
    "wide_range": dict(v_posed=1.2e-5, verts=3e-6, e2e=1.4e-5),
}


# ---------------------------------------------------------------------------------------------------------------------
# workspace layout, references and bounds (pure torch: shared by the GPU checks and the CPU calibration)
# ---------------------------------------------------------------------------------------------------------------------
def decode_workspace(ws, cap):
    """Views into an SMPL workspace of capacity `cap`, as laid out in romp_b200/csrc/smpl.cu:30-37: `cap` records of 736
    floats - [0,224) features, [224,512) A[24][3x4], [512,736) 448 fp16 = [hi(224) | lo(224)] of the features - then
    v_posed coordinate-tile major, [81][cap][256] floats."""
    flat = ws.reshape(-1)
    rec = flat[:cap * 736].view(cap, 736)
    tiles = flat[cap * 736:cap * 736 + 81 * cap * 256].view(81, cap, 256)
    return {"feat": rec[:, :224], "A": rec[:, 224:512].view(cap, NJ, 3, 4), "split": rec[:, 512:736], "tiles": tiles}


def v_posed_rows(tiles, c0, c1):
    """v_posed [c1-c0, 6890, 3] of persons c0..c1 from the coordinate-tile-major buffer"""
    return tiles[:, c0:c1].permute(1, 0, 2).reshape(c1 - c0, 81 * 256)[:, :COLS].reshape(c1 - c0, V, 3)


def blend_matrix(pack, n_betas, shape_key, device="cpu", dtype=torch.float64):
    """[K, 20670]: shapedirs rows (one per beta) then posedirs, the right operand of the blend GEMM"""
    s = torch.as_tensor(np.asarray(pack[shape_key])).to(device=device, dtype=dtype).reshape(COLS, n_betas).T
    return torch.cat([s, torch.as_tensor(np.asarray(pack["posedirs"])).to(device=device, dtype=dtype)])


def split_gemm_bound(a, b, k):
    """Per-element bound of a @ b (float64 tensors holding fp32 values, reduction length k) computed as hi hi' + lo hi' + hi lo'
    of the fp16 split with fp32 accumulation -> (bound, S = |a| @ |b|)."""
    aa, ba = a.abs(), b.abs()
    S = aa @ ba
    sub = SUBNORMAL * (aa.sum(-1, keepdim=True) + ba.sum(-2, keepdim=True))
    return (SPLIT_REL + U_TC * (3 * k + 3)) * S + sub, S


def blend_reference(f, B, vt):
    """v_posed = v_template + f B (f [n,K], B [K,20670], vt [20670]; float64) -> (value [n,20670], bound)"""
    bound, S = split_gemm_bound(f, B, f.shape[1])
    return vt + f @ B, bound + U32 * (vt.abs() + S)


def skin_reference(W, A, p):
    """verts = (W A) [p; 1] (W [6890,24], A [n,24,3,4], p [n,6890,3]; float64) -> (value [n,6890,3], bound).  The transforms
    T = W A come from the split GEMM; T [p; 1] is four fp32 products and sums per coordinate."""
    n = A.shape[0]
    Ab = A.reshape(n, NJ, 12).permute(1, 0, 2).reshape(NJ, n * 12)
    T = (W @ Ab).view(V, n, 3, 4).permute(1, 0, 2, 3)
    eT, S = split_gemm_bound(W, Ab, NJ)
    eT = eT.view(V, n, 3, 4).permute(1, 0, 2, 3)
    S = S.view(V, n, 3, 4).permute(1, 0, 2, 3)
    ph = torch.cat([p, torch.ones_like(p[..., :1])], -1).unsqueeze(-2)          # [n,V,1,4]
    value = (T * ph).sum(-1)
    bound = (eT * ph.abs()).sum(-1) + 5 * U32 * ((S + eT) * ph.abs()).sum(-1)
    return value, bound


def split16(x, ftz=False):
    """fp16 hi / lo parts (as fp32) of fp32 x, as smpl_pose_kernel and smpl_create build them; ftz: lo flushed to zero where
    it is an fp16 subnormal"""
    hi = x.half().float()
    lo = (x - hi).half().float()
    if ftz:
        lo = torch.where(lo.abs() < 2.0 ** -14, torch.zeros_like(lo), lo)
    return hi, lo


def emulate_split_gemm(a, b, products=("hh", "lh", "hl"), ftz=False):
    """a @ b (fp32) as the sum of the chosen fp16 part products, each exact in fp32, accumulated in fp32"""
    ah, al = split16(a, ftz)
    bh, bl = split16(b, ftz)
    parts = {"hh": (ah, bh), "lh": (al, bh), "hl": (ah, bl)}
    out = torch.zeros(a.shape[0], b.shape[1])
    for p in products:
        out = out + parts[p][0] @ parts[p][1]
    return out


def edge_inputs(n, stride=10, seed=0):
    """betas [n, stride] and thetas [n, 72] cycling through the input edges, person i gets case (i + seed) % 7:
    0 zero betas and thetas; 1 thetas of 1e-9; 2 every joint rotated by +-pi about a coordinate axis; 3 thetas uniform in
    +-3 rad; 4 the same with one component at 2 pi + 0.1; 5 betas of +-5; 6 betas N(0,1), thetas N(0,0.4)."""
    g = torch.Generator().manual_seed(seed)
    betas = torch.randn(n, stride, generator=g)
    thetas = 0.4 * torch.randn(n, 72, generator=g)
    uni = torch.rand(n, 72, generator=g) * 6 - 3
    wrap = torch.rand(n, 72, generator=g) * 6 - 3
    wrap[torch.arange(n), torch.randint(0, 72, (n,), generator=g)] = 2 * math.pi + 0.1
    axis = torch.randint(0, 3, (n, NJ, 1), generator=g)
    sign = (torch.randint(0, 2, (n, NJ, 1), generator=g) * 2 - 1).float()
    pi = torch.zeros(n, NJ, 3).scatter_(2, axis, sign * math.pi).view(n, 72)
    big = 5.0 * (torch.randint(0, 2, (n, stride), generator=g) * 2 - 1).float()
    case = ((torch.arange(n) + seed) % 7)[:, None]
    betas = torch.where(case == 0, torch.zeros_like(betas), betas)
    betas = torch.where(case == 5, big, betas)
    thetas = torch.where(case == 0, torch.zeros_like(thetas), thetas)
    thetas = torch.where(case == 1, torch.full_like(thetas, 1e-9), thetas)
    thetas = torch.where(case == 2, pi, thetas)
    thetas = torch.where(case == 3, uni, thetas)
    thetas = torch.where(case == 4, wrap, thetas)
    return betas.contiguous(), thetas.contiguous()


def bench_inputs(n):
    """bench.py --workload smpl's inputs"""
    g = torch.Generator(device="cpu").manual_seed(0)
    betas = torch.randn(n, 10, generator=g)
    thetas = torch.randn(n, 72, generator=g) * 0.3
    return betas, thetas


# ---------------------------------------------------------------------------------------------------------------------
# the CPU calibration of the two checks
# ---------------------------------------------------------------------------------------------------------------------
BLEND_MUTANTS = {"f_lo*B_hi dropped": dict(products=("hh", "hl")), "f_hi*B_lo dropped": dict(products=("hh", "lh")),
                 "hi only": dict(products=("hh",)), "lo flushed when subnormal": dict(ftz=True)}
SKIN_MUTANTS = {"W_lo*A_hi dropped": dict(products=("hh", "hl")), "W_hi*A_lo dropped": dict(products=("hh", "lh")),
                "hi only": dict(products=("hh",)), "lo flushed when subnormal": dict(ftz=True)}


def _judge(got, ref, bound):
    err = (got.double() - ref).abs()
    return err.max().item(), (err / bound).max().item(), int((err > bound).sum())


@pytest.mark.parametrize("variant", synth.SMPL_PACK_VARIANTS)
def test_split_calibration_cpu(variant):
    """An emulation of the kernels' exact arithmetic (fp16 hi / lo parts, their three products exact in fp32, fp32
    accumulation) lies within the per-element bound and the global limit of both GEMM stages, and within the end-to-end
    limit; emulations that drop a cross term, keep hi only or flush subnormal lo parts to zero are rejected."""
    pack = synth.smpl_pack(0, variant=variant)
    lim = LIMITS[variant]
    betas, thetas = edge_inputs(28, seed=3)
    v64, j64, s64 = O.smpl_forward(pack, betas, thetas, dtype=torch.float64, stages=True)
    _, _, s32 = O.smpl_forward(pack, betas, thetas, stages=True)
    B32 = blend_matrix(pack, 10, "shapedirs", dtype=torch.float32)
    vt32 = torch.as_tensor(pack["v_template"]).reshape(-1)
    W32 = torch.as_tensor(pack["weights"])
    f32, A32 = s32["feat"], s32["A"]                       # the fp32 stages the GPU's pose kernel would hand on
    n = f32.shape[0]
    Ab32 = A32.reshape(n, NJ, 12).permute(1, 0, 2).reshape(NJ, n * 12)
    vref, vbound = blend_reference(f32.double(), B32.double(), vt32.double())

    def blend(**kw):
        return vt32 + emulate_split_gemm(f32, B32, **kw)

    def skin(p, **kw):
        T = emulate_split_gemm(W32, Ab32, **kw).view(V, n, 3, 4).permute(1, 0, 2, 3)
        return T[..., 0] * p[..., 0:1] + T[..., 1] * p[..., 1:2] + T[..., 2] * p[..., 2:3] + T[..., 3]

    vp = blend()
    e, r, over = _judge(vp, vref, vbound)
    print(f"\n{variant}: emulated split  v_posed max|err| {e:.2e} (limit {lim['v_posed']:.0e}) max err/bound {r:.3f}")
    assert over == 0 and e <= lim["v_posed"]
    p = vp.view(n, V, 3)
    sref, sbound = skin_reference(W32.double(), A32.double(), p.double())
    verts = skin(p)
    e, r, over = _judge(verts, sref, sbound)
    print(f"{variant}: emulated split  verts   max|err| {e:.2e} (limit {lim['verts']:.0e}) max err/bound {r:.3f}")
    assert over == 0 and e <= lim["verts"]
    e2e = (verts.double() - v64).abs().max().item()
    o32 = (O.smpl_forward(pack, betas, thetas)[0].double() - v64).abs().max().item()
    print(f"{variant}: emulated split  e2e verts max|err| {e2e:.2e} (limit {lim['e2e']:.0e}; fp32 oracle {o32:.2e})")
    assert e2e <= lim["e2e"]

    for name, kw in BLEND_MUTANTS.items():
        e, r, over = _judge(blend(**kw), vref, vbound)
        print(f"{variant}: {name:26s} v_posed max|err| {e:.2e} max err/bound {r:8.2f} ({over} elements over)")
        assert e > 3 * lim["v_posed"], f"{name}: global limit accepts it"
        assert over > 0, f"{name}: per-element bound accepts it"
    for name, kw in SKIN_MUTANTS.items():
        e, r, over = _judge(skin(p, **kw), sref, sbound)
        print(f"{variant}: {name:26s} verts   max|err| {e:.2e} max err/bound {r:8.2f} ({over} elements over)")
        assert e > 3 * lim["verts"], f"{name}: global limit accepts it"
        assert over > 0, f"{name}: per-element bound accepts it"


def test_edge_inputs_cover_the_cases():
    betas, thetas = edge_inputs(14, seed=0)
    t = thetas.view(14, NJ, 3)
    assert (betas[0] == 0).all() and (thetas[0] == 0).all()
    assert (thetas[1] == np.float32(1e-9)).all()
    assert ((t[2].abs() == np.float32(math.pi)).sum(1) == 1).all() and ((t[2] == 0).sum(1) == 2).all()
    assert thetas[3].abs().max() <= 3 and (thetas[4] == np.float32(2 * math.pi + 0.1)).sum() == 1
    assert (betas[5].abs() == 5).all()
    # the split variants keep the default pack as it was
    d, r = synth.smpl_pack(0), synth.smpl_pack(0, variant="real_scale")
    assert all(np.array_equal(d[k], r[k]) for k in d if k not in ("shapedirs", "posedirs"))
    w = synth.smpl_pack(0, variant="wide_range")["weights"]
    assert np.allclose(w.sum(1), 1, atol=1e-6) and w.min() > 0 and np.sort(w, 1)[:, -2].max() <= 0.1


# ---------------------------------------------------------------------------------------------------------------------
# the GPU run, checked stage by stage
# ---------------------------------------------------------------------------------------------------------------------
class Stats:
    def __init__(self):
        self.pose, self.gemm, self.e2e = {}, {}, {}

    def add_pose(self, stage, got, r64, r32):
        e, e32, m = self.pose.get(stage, (0.0, 0.0, 0.0))
        self.pose[stage] = (max(e, (got.double() - r64).abs().max().item()), max(e32, (r32.double() - r64).abs().max().item()),
                            max(m, r64.abs().max().item()))

    def add_gemm(self, stage, got, ref, bound):
        err = (got.double() - ref).abs()
        e, r, over = self.gemm.get(stage, (0.0, 0.0, 0))
        self.gemm[stage] = (max(e, err.max().item()), max(r, (err / bound).max().item()), over + int((err > bound).sum()))

    def add_e2e(self, stage, got, ref):
        self.e2e[stage] = max(self.e2e.get(stage, 0.0), (got.double() - ref).abs().max().item())

    def report(self, label, lim):
        bad = []
        for stage, (e, e32, m) in self.pose.items():
            allowed = POSE_FACTOR * e32 + POSE_FLOOR * max(1.0, m)
            print(f"  {label}  pose {stage:11s} max|err| {e:.2e}  fp32 oracle {e32:.2e}  allowed {allowed:.2e}")
            if e > allowed:
                bad.append(f"pose {stage}: {e:.2e} > {allowed:.2e}")
        for stage, (e, r, over) in self.gemm.items():
            L = lim.get(stage)
            print(f"  {label}  {stage:16s} max|err| {e:.2e}  max err/bound {r:.3f}" + (f"  limit {L:.1e}" if L else ""))
            if over:
                bad.append(f"{stage}: {over} elements over the bound (max err/bound {r:.3f})")
            if L is not None and e > L:
                bad.append(f"{stage}: max|err| {e:.2e} > limit {L:.1e}")
        for stage, e in self.e2e.items():
            print(f"  {label}  end-to-end {stage:6s} max|err| {e:.2e}  limit {lim['e2e']:.1e}")
            if e > lim["e2e"]:
                bad.append(f"end-to-end {stage}: {e:.2e} > {lim['e2e']:.1e}")
        assert not bad, f"{label}: " + "; ".join(bad)


class Smpl:
    """One SMPL model: the GPU kernels (SMPLParser) and float64 copies of its matrices on the device"""

    def __init__(self, pack, kind="synthetic", n_betas=10, shape_key="shapedirs"):
        from romp_b200.main import SMPLParser
        self.sm = SMPLParser(pack, 0, n_betas=n_betas, shape_key=shape_key)
        self.pack, self.kind, self.nb, self.K, self.key = pack, kind, n_betas, n_betas + 207, shape_key
        d = lambda k: torch.as_tensor(np.asarray(pack[k])).to(device=DEV, dtype=torch.float64)
        self.B = blend_matrix(pack, n_betas, shape_key, DEV)
        self.vt = d("v_template").reshape(-1)
        self.W = d("weights")
        self.jreg = torch.cat([d("J_regressor_extra9"), d("J_regressor_h36m17")])
        self.jreg_bound = U32 * ((self.jreg != 0).sum(1, keepdim=True) + 6) * 1.0
        self.extra = torch.as_tensor(np.asarray(pack["extra_joints_index"]), device=DEV)

    def run(self, betas, thetas, cap, count, root_align):
        verts = torch.full((cap, V, 3), SENTINEL, device=DEV)
        joints = torch.full((cap, 71, 3), SENTINEL, device=DEV)
        ws = torch.zeros(cap, self.sm.ws_floats, device=DEV)
        cnt = None if count is None else torch.tensor([count], dtype=torch.int32, device=DEV)
        self.sm.forward(betas, thetas, cap, cnt, root_align, ws, verts, joints, torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        n = cap if count is None else max(0, min(count, cap))
        assert (verts[n:] == SENTINEL).all() and (joints[n:] == SENTINEL).all(), "rows at or past the count were written"
        return n, verts, joints, ws

    def check(self, label, betas, thetas, cap, count=None, root_align_too=False):
        """One forward without root_align, every stage checked; with root_align_too a second, aligned forward checked bit for
        bit against the first.  betas / thetas: CPU tensors of `cap` rows."""
        t0 = time.time()
        b, t = betas.to(DEV), thetas.to(DEV)
        n, verts, joints, ws = self.run(b, t, cap, count, False)
        stats = Stats()
        wsv = decode_workspace(ws, cap)
        for c0 in range(0, n, CHUNK):
            self._check_chunk(stats, wsv, b, t, verts, joints, c0, min(n, c0 + CHUNK))
        print(f"{label}: capacity {cap}, count {count}, {n} persons checked in {time.time() - t0:.1f} s")
        if n:
            stats.report(label, LIMITS[self.kind])
        del ws, wsv
        if root_align_too:
            n2, verts_ra, joints_ra, ws_ra = self.run(b, t, cap, count, True)
            root = (joints[:n, 45] + joints[:n, 46]) / 2                       # fp32, like smpl_joints_kernel
            assert torch.equal(decode_workspace(ws_ra, cap)["feat"][:n, :3], root), "root"
            assert torch.equal(joints_ra[:n], joints[:n] - root[:, None]), "root-aligned joints"
            assert torch.equal(verts_ra[:n], verts[:n] - root[:, None]), "root-aligned verts"
            print(f"  {label}  root_align: root and subtraction bit-exact")

    def _check_chunk(self, stats, wsv, b, t, verts, joints, c0, c1):
        nb, K = self.nb, self.K
        bb, tt = b[c0:c1, :nb], t[c0:c1]
        feat, A = wsv["feat"][c0:c1, :K], wsv["A"][c0:c1]
        # pose kernel: the features start with the betas; the fp16 split is exact
        assert torch.equal(feat[:, :nb], bb), "features: betas"
        f224 = torch.zeros(c1 - c0, 224, device=DEV)
        f224[:, :K] = feat
        hi = f224.half()
        split = wsv["split"][c0:c1].contiguous().view(torch.float16)
        assert torch.equal(split[:, :224], hi) and torch.equal(split[:, 224:], (f224 - hi.float()).half()), "fp16 split"
        v64, j64, s64 = O.smpl_forward(self.pack, bb, tt, shape_key=self.key, dtype=torch.float64, device=DEV, stages=True)
        v32, j32, s32 = O.smpl_forward(self.pack, bb, tt, shape_key=self.key, device=DEV, stages=True)
        stats.add_pose("features", feat, s64["feat"], s32["feat"])
        stats.add_pose("A", A, s64["A"], s32["A"])
        stats.add_pose("joints0-23", joints[c0:c1, :NJ], j64[:, :NJ], j32[:, :NJ])
        del v32, j32, s32, s64
        # blend GEMM on the GPU's features
        vp = v_posed_rows(wsv["tiles"], c0, c1)
        ref, bound = blend_reference(feat.double(), self.B, self.vt)
        stats.add_gemm("v_posed", vp.reshape(c1 - c0, COLS), ref, bound)
        del ref, bound
        # skinning GEMM on the GPU's A and v_posed
        vg = verts[c0:c1]
        ref, bound = skin_reference(self.W, A.double(), vp.double())
        stats.add_gemm("verts", vg, ref, bound)
        del ref, bound
        # joints kernel on the GPU's verts
        jg = joints[c0:c1]
        assert torch.isfinite(vg).all() and torch.isfinite(jg).all()
        assert torch.equal(jg[:, 24:45], vg[:, self.extra]), "joints 24-44 are not the picked vertices"
        vd = vg.double()
        ref = torch.einsum("rv,nvk->nrk", self.jreg, vd)
        bound = self.jreg_bound[None] * torch.einsum("rv,nvk->nrk", self.jreg.abs(), vd.abs())
        stats.add_gemm("joints45-70", jg[:, 45:], ref, bound)
        stats.add_e2e("verts", vg, v64)
        stats.add_e2e("joints", jg, j64)


_MODELS = {}


def model(name):
    """the Smpl models of the tests, built once per session"""
    if name not in _MODELS:
        kind, nb, key, pack = {
            "synthetic": ("synthetic", 10, "shapedirs", lambda: synth.smpl_pack(0)),
            "real_scale": ("real_scale", 10, "shapedirs", lambda: synth.smpl_pack(0, variant="real_scale")),
            "wide_range": ("wide_range", 10, "shapedirs", lambda: synth.smpl_pack(0, variant="wide_range")),
            "betas1": ("synthetic", 1, "smpla_shapedirs", lambda: synth.smpl_pack(0, num_betas=1)),
            "betas16": ("synthetic", 16, "smpla_shapedirs", lambda: synth.smpl_pack(0, num_betas=16)),
            "smpla": ("synthetic", 11, "smpla_shapedirs", lambda: synth.smpl_pack(0, num_betas=11)),
            "smil": ("synthetic", 10, "shapedirs", lambda: synth.smpl_pack(1)),
        }[name]
        _MODELS[name] = Smpl(pack(), kind, nb, key)
    return _MODELS[name]


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 127, 128, 129, 300])
def test_tile_edges(n):
    """person counts at the blend GEMM's 128-person tiles and the skinning GEMM's 8-person tiles, every input edge"""
    betas, thetas = edge_inputs(n, seed=n)
    model("synthetic").check(f"tile edge n={n}", betas, thetas, n, root_align_too=True)


@pytest.mark.gpu
@pytest.mark.parametrize("count", [0, 1, 9, 129, 4096, 4100])
def test_romp_capacity_device_count(count):
    """ROMP's production call: capacity 64 x batch 64 = 4096 with the person count on the device (clamped to the capacity)"""
    betas, thetas = edge_inputs(4096, seed=count)
    model("synthetic").check(f"ROMP cap 4096 count {count}", betas, thetas, 4096, count)


@pytest.mark.gpu
def test_skinning_ctas_loop():
    """5,000 persons: 625 skinning tiles on at most 4 x SMs CTAs, so CTAs loop over person tiles"""
    betas, thetas = edge_inputs(5000, seed=5000)
    model("synthetic").check("skinning loop n=5000", betas, thetas, 5000, root_align_too=True)


@pytest.mark.gpu
def test_benchmark_persons():
    """bench.py --workload smpl: 65,536 persons with its inputs, every person checked stage-wise"""
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.time()
    betas, thetas = bench_inputs(65536)
    model("synthetic").check("benchmark n=65536", betas, thetas, 65536)
    print(f"benchmark n=65536: {time.time() - t0:.1f} s, peak torch allocation {torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB")


@pytest.mark.gpu
@pytest.mark.parametrize("n_betas", [1, 16])
def test_n_betas(n_betas):
    """K = n_betas + 207 from 208 to 223 (one pad column left in the 224-wide operand)"""
    betas, thetas = edge_inputs(300, stride=n_betas, seed=n_betas)
    model(f"betas{n_betas}").check(f"n_betas {n_betas}", betas, thetas, 300, 261, root_align_too=True)


@pytest.mark.gpu
@pytest.mark.parametrize("variant", ["real_scale", "wide_range"])
def test_packs(variant):
    """the released model's magnitudes, and blend entries / skinning weights spanning 1e-8 to 1e-1"""
    betas, thetas = edge_inputs(300, seed=7)
    model(variant).check(f"{variant} pack", betas, thetas, 300, 261, root_align_too=True)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["smpla", "smil"])
def test_bev_models(name):
    """BEV's production call: capacity 32 x 64 = 2048 with a device count and root_align, on the shared [cap, 11] betas
    (SMPL-A reads 11 betas, SMIL the first 10 at stride 11)"""
    betas, thetas = edge_inputs(2048, stride=11, seed=11)
    model(name).check(f"BEV {name}", betas, thetas, 2048, 1999, root_align_too=True)


@pytest.mark.gpu
def test_bev_smil_merge_threshold():
    """BEV's run_post takes SMIL's mesh exactly for the rows with betas[:, 10] > 0.8 (bev/post_parser.py:260-263),
    at 0.8f, the next float above it and 0.7999"""
    from romp_b200.bev import BEV, bev_settings
    s = bev_settings(["--precision", "fp32", "--max_batch", "32"])
    m = BEV(s, state_dict=synth.bev_state_dict(0), smpla_pack=synth.smpl_pack(0, num_betas=11), smil_pack=synth.smpl_pack(1))
    cap, n = m.cap, 1999
    assert cap == 2048
    betas, thetas = edge_inputs(cap, stride=11, seed=12)
    g = torch.Generator().manual_seed(13)
    betas[:, 10] = 0.6 + 0.4 * torch.rand(cap, generator=g)
    edge = np.array([0.8, np.nextafter(np.float32(0.8), np.float32(1)), 0.7999], np.float32)
    betas[:3, 10] = torch.from_numpy(edge)
    b = m.buf
    b["betas"].copy_(betas)
    b["thetas"].copy_(thetas)
    b["cam"].copy_(torch.tensor([0.5, 0.0, 0.0]).expand(cap, 3))
    b["cam_trans"].copy_(torch.tensor([0.0, 0.0, 5.0]).expand(cap, 3))
    b["batch_ids"].copy_(torch.arange(cap) // 64)
    b["count"][0] = n
    with torch.cuda.stream(m.stream):
        m.run_post(32, [0, 512, 0, 512, 512, 512], 512.0)
    m.stream.synchronize()
    va = torch.full((cap, V, 3), SENTINEL, device=DEV)
    ja = torch.full((cap, 71, 3), SENTINEL, device=DEV)
    ws = torch.zeros(cap, m.smpla.ws_floats, device=DEV)
    m.smpla.forward(b["betas"], b["thetas"], cap, b["count"], True, ws, va, ja, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    baby = torch.from_numpy(betas[:n, 10].numpy() > np.float32(0.8)).to(DEV)
    assert baby[:3].tolist() == [False, True, False] and 0 < int(baby.sum()) < n
    vs, js = b["verts_smil"][:n], b["joints_smil"][:n]
    assert not torch.equal(vs[baby], va[:n][baby])                           # the two models differ on these rows
    assert torch.equal(b["verts"][:n][baby], vs[baby]) and torch.equal(b["joints"][:n][baby], js[baby])
    assert torch.equal(b["verts"][:n][~baby], va[:n][~baby]) and torch.equal(b["joints"][:n][~baby], ja[:n][~baby])
    print(f"BEV merge: {int(baby.sum())} of {n} rows from SMIL, the rest SMPL-A, bit for bit")
