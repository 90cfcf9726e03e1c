"""BEV detection stages between the conv graphs and SMPL-A (romp_b200/csrc/bev.cu), each run through the C ABI on its own
device inputs and compared with a float64 restatement built from the UNFOLDED state dict (so the BatchNorm3d folding of
graph.bev_weights is checked too):
  bev_bv_input               bit-exact against torch.cat(...).view(B, 2560, 128)
  bev_center3d (fused)       every voxel against fp64 block_3d(fv (x) bv), per-voxel error bound
  bev_parse3d                bit-exact against bev_oracle.parse_3d at its edges, and past 4096 local maxima per frame
  bev_regress + bev_unpack   cams against the full-volume fp64 cam refiner, cam_czyx, MLP and unpack against fp64
Inputs are what BEV.run_model leaves in m.buf for synthetic frames (fp32 and bf16 graphs), and crafted tensors with a
wide dynamic range and energy on the volume faces and the 8 x 8 x 32 tile seams of the fused centre kernel.

Error bounds are per element, |err| <= gamma * 2^-24 * cond + tiny, where cond is the same restatement run on |weights|
and |inputs| with ReLU replaced by the identity (an upper bound on every partial sum the fp32 kernel rounds)."""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import bev_oracle as B
from oracle import romp_oracle as O
from romp_b200 import _lib, graph, synth
from romp_b200._lib import BF16, F32
from romp_b200.bev import BEV, bev_settings

pytestmark = pytest.mark.gpu
P = lambda t: C.c_void_p(t.data_ptr())
U = 2.0 ** -24
TINY = 1e-30
G_CENTER, G_CAM, G_MLP = 32.0, 64.0, 64.0
SENT = -7
THRESH = 0.08
DEV = "cuda"
ACT = {"fp32": (torch.float32, F32), "bf16": (torch.bfloat16, BF16)}
_models = {}


def stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


@pytest.fixture(scope="module")
def sd():
    return synth.bev_state_dict(0)


@pytest.fixture(scope="module")
def sd64(sd):
    keep = ("center_map_refiner.", "cam_map_refiner.", "transformer.", "position_embeddings.", "coordmap_3d")
    return {k: torch.from_numpy(np.asarray(v)).to(DEV, torch.float64) for k, v in sd.items() if k.startswith(keep)}


def model(sd, precision):
    """BEV at max_batch 32 without SMPL: its handle (m.h) carries the folded weights the kernels read."""
    if precision not in _models:
        s = bev_settings(["--precision", precision, "--max_batch", "32", "--calc_smpl"])
        _models[precision] = BEV(s, state_dict=sd)
    return _models[precision]


@pytest.fixture(scope="module", params=["fp32", "bf16"])
def model_state(request, sd):
    """m after run_model on 3 synthetic frames: m.buf holds maps_fv, bv_in, bv_out, img_feats, fv_feats, center3d."""
    m = model(sd, request.param)
    frames = torch.from_numpy(synth.synthetic_frames(3, seed=11)).to(DEV)
    with torch.cuda.stream(m.stream):
        m.run_model(frames)
    m.stream.synchronize()
    return request.param, m


# ------------------------------------------------------------------------------------------------ fp64 restatements
def block_3d_abs(sd64, p, x):
    """cond of B.block_3d: |BN scale| * conv(|w|, x) + |BN shift| per stage (ReLU -> identity), plus the residual x;
    x is the |input| bound."""
    def stage(i, x):
        s = sd64[f"{p}bn{i}.weight"] / torch.sqrt(sd64[f"{p}bn{i}.running_var"] + O.BN_EPS)
        shift = sd64[f"{p}bn{i}.bias"] - sd64[f"{p}bn{i}.running_mean"] * s
        y = F.conv3d(x, sd64[f"{p}conv{i}.weight"].abs(), None, 1, 1)
        return y * s.abs().view(1, -1, 1, 1, 1) + shift.abs().view(1, -1, 1, 1, 1)
    return stage(2, stage(1, x)) + x


def center3d_fp64(sd64, maps_fv, bv):
    """(value, cond) [B,64,128,128] of refiner(center_fv (x) center_bv), bev/model.py:195-196,206."""
    n = maps_fv.shape[0]
    cfv = maps_fv[:, 0].double()                                          # [B,h,w]
    cbv = bv.reshape(n, 128, 128)[:, :, :64].double().permute(0, 2, 1)    # [B,d,w]
    cm = cfv[:, None] * cbv[:, :, None, :]
    ref = B.block_3d(sd64, "center_map_refiner.0.", cm[:, None])[:, 0]
    cond = block_3d_abs(sd64, "center_map_refiner.0.", cm.abs()[:, None])[:, 0]
    return ref, cond


def cam_volume_fp64(sd64, maps_fv_b, bv_b):
    """(value, cond) [3,64,128,128] of the cam refiner over the whole volume of one frame, bev/model.py:209-213."""
    cmap = sd64["coordmap_3d"][0]                                         # [d,h,w,3]
    off = maps_fv_b[1:4].double().permute(1, 2, 0)[None]                  # [1,h,w,3]
    obv = bv_b.reshape(128, 128)[:, 64:].double().T[:, None, :]           # [d,1,w]
    x = cmap + off
    x[..., 2] += obv
    xa = cmap.abs() + off.abs()
    xa[..., 2] += obv.abs()
    ref = B.block_3d(sd64, "cam_map_refiner.0.", x.permute(3, 0, 1, 2)[None])[0]
    cond = block_3d_abs(sd64, "cam_map_refiner.0.", xa.permute(3, 0, 1, 2)[None])[0]
    return ref, cond


def check_bound(name, got, ref, cond, gamma):
    err = (got.double() - ref).abs()
    bound = gamma * U * cond + TINY
    ratio = (err / bound).max().item()
    print(f"{name}: max|err| {err.max().item():.3e}  worst err/bound {ratio:.3f} (gamma {gamma:g})")
    bad = torch.nonzero(~(err <= bound))                   # NaN (an unwritten or garbage element) fails too
    assert len(bad) == 0, f"{name}: {len(bad)} elements outside the bound or not finite, first {bad[:5].tolist()}"
    assert ratio <= 1.0
    return ratio


# ------------------------------------------------------------------------------------------------ kernel calls
def run_bv_input(maps_fv, feats, code):
    n = maps_fv.shape[0]
    out = torch.full((n, 1, 128, 2560), float("nan"), dtype=feats.dtype, device=DEV)
    _lib.check(_lib.load().b200romp_bev_bv_input(P(maps_fv), P(feats), code, feats.shape[-1], n, P(out), code, stream()), "bv_input")
    torch.cuda.synchronize()
    return out


def run_center3d(m, maps_fv, bv, code):
    n = maps_fv.shape[0]
    out = torch.full((n, 64, 128, 128), float("nan"), device=DEV)
    _lib.check(m.lib.b200romp_bev_center3d(m.h, P(maps_fv), P(bv), code, n, P(m.buf["c3d_tmp"]), P(out), stream()), "center3d")
    torch.cuda.synchronize()
    return out


def run_parse(vol, thresh=THRESH, cap=None):
    """-> (count, batch_ids, czyx, conf) on the host; rows past the count must keep their sentinel."""
    lib, n = _lib.load(), vol.shape[0]
    cap = cap or n * 64
    ws = torch.zeros(int(lib.b200romp_bev_parse_workspace_bytes(n)), dtype=torch.uint8, device=DEV)
    cnt = torch.full((1,), SENT, dtype=torch.int32, device=DEV)
    bi = torch.full((cap,), SENT, dtype=torch.int64, device=DEV)
    czyx = torch.full((cap, 3), SENT, dtype=torch.int64, device=DEV)
    conf = torch.full((cap,), SENT, dtype=torch.float32, device=DEV)
    _lib.check(lib.b200romp_bev_parse3d(P(vol), n, float(thresh), cap, P(cnt), P(bi), P(czyx), P(conf), P(ws), stream()), "parse3d")
    torch.cuda.synchronize()
    k = int(cnt.item())
    assert (bi[k:] == SENT).all() and (czyx[k:] == SENT).all() and (conf[k:] == SENT).all()
    return k, bi[:k].cpu().numpy(), czyx[:k].cpu().numpy(), conf[:k].cpu().numpy()


def assert_parse_exact(vol_np, thresh=THRESH, cap=None, gpu=None):
    """GPU parse (or the given GPU rows) == bev_oracle.parse_3d (value desc, voxel index asc), bit for bit; returns the
    GPU rows."""
    k, bi, czyx, conf = gpu or run_parse(torch.from_numpy(vol_np).to(DEV), thresh, cap)
    rb, rz, rc = B.parse_3d(vol_np, thresh)
    want = len(rb) if cap is None else min(len(rb), cap)
    assert k == want
    assert np.array_equal(bi, rb.numpy()[:k]) and np.array_equal(czyx, rz.numpy()[:k]) and np.array_equal(conf, rc.numpy()[:k])
    return bi, czyx, conf


def run_regress(m, maps_fv, bv, fv, code, count, bi, czyx, cap):
    o = dict(pp=(cap, 146), cc=(cap, 3), cam=(cap, 3), th=(cap, 72), be=(cap, 11), tr=(cap, 3))
    o = {k: torch.full(s, SENT, dtype=torch.int64 if k == "cc" else torch.float32, device=DEV) for k, s in o.items()}
    d_count = count if isinstance(count, torch.Tensor) else torch.tensor([count], dtype=torch.int32, device=DEV)
    _lib.check(m.lib.b200romp_bev_regress(m.h, P(maps_fv), P(bv), code, P(fv), code, cap, P(d_count), P(bi), P(czyx),
                                          P(o["pp"]), P(o["cc"]), P(o["cam"]), P(o["th"]), P(o["be"]), P(o["tr"]), stream()),
               "regress")
    torch.cuda.synchronize()
    n = int(d_count.item())
    for k, v in o.items():
        assert (v[n:] == SENT).all(), f"regress wrote {k} rows past the count"
    return n, {k: v[:n] for k, v in o.items()}


# ------------------------------------------------------------------------------------------------ crafted inputs
FACE = [0, 1, 2, 125, 126, 127]
SEAM_HW = sorted({0, 127} | {w for w in range(128) if w % 32 in (0, 31)})     # faces and tile seams along w
SEAM_H = sorted({0, 127} | {h for h in range(128) if h % 8 in (0, 7)})
SEAM_D = sorted({0, 63} | {d for d in range(64) if d % 8 in (0, 7)})


def crafted_maps(n, seed, dtype):
    """maps_fv [n,4,128,128] fp32, bv_out [n,1,128,128] and fv_feats [n,128,128,128] in `dtype`: magnitudes over four
    decades, centre energy x100 on the faces and tile seams of h, w and d."""
    g = torch.Generator().manual_seed(seed)
    wide = lambda *s: torch.randn(*s, generator=g) * 10.0 ** (torch.rand(*s, generator=g) * 4 - 2)
    maps_fv = wide(n, 4, 128, 128)
    maps_fv[:, 1:4] = torch.randn(n, 3, 128, 128, generator=g) * 0.3               # cam offsets of a plausible size
    maps_fv[:, 0, SEAM_H] *= 100.0
    maps_fv[:, 0, :, SEAM_HW] *= 100.0
    bv = wide(n, 128, 128)                                                          # [b, w, channel]
    bv[:, :, 64:] = torch.randn(n, 128, 64, generator=g) * 0.3
    bv[:, SEAM_HW, :64] *= 100.0
    bv[:, :, SEAM_D] *= 100.0
    fv = torch.randn(n, 128, 128, 128, generator=g)
    return maps_fv.to(DEV), bv.reshape(n, 1, 128, 128).to(DEV, dtype), fv.to(DEV, dtype)


# ================================================================================================ bv_input
def bv_input_ref(maps_fv, feats, dtype):
    """torch.cat([center_fv, cam_off, img_feats[..., :16]], 1).view(B, 2560, 128) in the kernel's [B, 128(w), 2560]."""
    n = maps_fv.shape[0]
    cat = torch.cat([maps_fv, feats[..., :16].permute(0, 3, 1, 2).float()], 1).reshape(n, 2560, 128)
    return cat.transpose(1, 2).contiguous().to(dtype).reshape(n, 1, 128, 2560)


def bits(t):
    return t.view(torch.int16 if t.dtype == torch.bfloat16 else torch.int32)


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("batch", [1, 32])
def test_bv_input_bit_exact(precision, batch):
    dtype, code = ACT[precision]
    g = torch.Generator().manual_seed(batch)
    maps_fv = (torch.randn(batch, 4, 128, 128, generator=g) * 10.0 ** (torch.rand(batch, 4, 128, 128, generator=g) * 8 - 4)).to(DEV)
    cf = graph.bev_feats_channels(precision)
    feats = torch.randn(batch, 128, 128, cf, generator=g).to(DEV, dtype)
    out = run_bv_input(maps_fv, feats, code)
    assert torch.equal(bits(out), bits(bv_input_ref(maps_fv, feats, dtype)))


def test_bv_input_model_state(model_state):
    precision, m = model_state
    b, n = m.buf, 3
    dtype, code = ACT[precision]
    assert torch.equal(bits(b["bv_in"][:n]), bits(bv_input_ref(b["maps_fv"][:n], b["img_feats"][:n], dtype)))
    out = run_bv_input(b["maps_fv"][:n].contiguous(), b["img_feats"][:n].contiguous(), code)
    assert torch.equal(bits(out), bits(b["bv_in"][:n]))


# ================================================================================================ center3d
def check_center3d(m, sd64, maps_fv, bv, code, name):
    out = run_center3d(m, maps_fv, bv, code)
    worst = 0.0
    for c0 in range(0, maps_fv.shape[0], 8):                                        # 8 frames of fp64 at a time
        ref, cond = center3d_fp64(sd64, maps_fv[c0:c0 + 8], bv[c0:c0 + 8])
        worst = max(worst, check_bound(f"{name} frames {c0}..", out[c0:c0 + 8], ref, cond, G_CENTER))
    print(f"center3d {name}: worst err/bound {worst:.3f}")
    return out


def test_center3d_model_state(model_state, sd64):
    precision, m = model_state
    b, n = m.buf, 3
    out = check_center3d(m, sd64, b["maps_fv"][:n], b["bv_out"][:n], ACT[precision][1], f"model {precision}")
    assert torch.equal(out, b["center3d"][:n])                                     # the same kernel run_model launched


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("batch", [1, 3, 32])
def test_center3d_crafted(sd, sd64, precision, batch):
    m = model(sd, precision)
    maps_fv, bv, _ = crafted_maps(batch, 100 + batch, ACT[precision][0])
    check_center3d(m, sd64, maps_fv, bv, ACT[precision][1], f"crafted {precision} B={batch}")


# ================================================================================================ parse3d
def plant(vol, cells):
    for (z, y, x), v in cells:
        vol[z, y, x] = np.float32(v)


def random_peaks(rs, n, lo=0.25, hi=1.0, sep=3):
    """n cells at random positions (all depths), pairwise Chebyshev distance >= sep, with distinct values in (lo, hi)."""
    cells = []
    while len(cells) < n:
        c = (rs.randint(0, 64), rs.randint(0, 128), rs.randint(0, 128))
        if all(max(abs(c[0] - q[0]), abs(c[1] - q[1]), abs(c[2] - q[2])) >= sep for q in cells):
            cells.append(c)
    vals = lo + (hi - lo) * rs.permutation(n) / n
    return list(zip(cells, vals))


def lattice_peaks(rs, n, lo=0.25, hi=1.0, levels=None):
    """n distinct cells of the 3-spaced lattice (so no two suppress each other), values in (lo, hi): all distinct, or
    drawn from `levels` equal values (ties)."""
    lat = np.stack(np.meshgrid(np.arange(0, 64, 3), np.arange(0, 128, 3), np.arange(0, 128, 3), indexing="ij"), -1).reshape(-1, 3)
    cells = lat[rs.choice(len(lat), n, replace=False)]
    k = rs.permutation(n) if levels is None else rs.randint(0, levels, n)
    vals = lo + (hi - lo) * k / (n if levels is None else levels)
    return [(tuple(c), v) for c, v in zip(cells.tolist(), vals)]


def dense_frame(seed, n_peaks=80):
    """bev_noise_volume (> 4096 local maxima) with n_peaks planted above the noise at random depths."""
    vol = synth.bev_noise_volume(seed)[0]
    plant(vol, random_peaks(np.random.RandomState(seed), n_peaks))
    return vol


def tie_frame(seed):
    """noise on a grid of 1e-6 steps: ~10 voxels per level at the top, so the top-64 spans levels with ties inside each."""
    rs = np.random.RandomState(seed)
    return (0.1 + 1e-6 * rs.randint(0, 100000, size=(64, 128, 128))).astype(np.float32)


def edge_batch():
    """32 frames, one parse edge each (frames 15.. dense); returns (vol, names)."""
    rs = np.random.RandomState(4)
    vol = np.zeros((32, 64, 128, 128), np.float32)
    names = {}
    vol[0] = rs.uniform(0, 0.05, size=(64, 128, 128))                                 # sparse planted peaks on low noise
    plant(vol[0], random_peaks(rs, 6, 0.2, 1.0))
    names[0] = "sparse"
    plant(vol[1], [((10, 20, 30), 0.5), ((10, 20, 31), 0.5), ((40, 90, 7), 0.5), ((41, 90, 7), 0.5)])   # equal adjacent maxima
    names[1] = "equal adjacent"
    pairs = []                                                                          # 2 apart: suppressed, 3 apart: kept
    for i, (dz, dy, dx) in enumerate(((1, 0, 0), (0, 1, 0), (0, 0, 1), (1, 1, 1))):
        for j, dist in enumerate((2, 3)):
            z, y, x = 6 + 12 * i, 10 + 30 * j, 64
            pairs += [((z, y, x), 0.9 - 0.05 * (2 * i + j)), ((z + dist * dz, y + dist * dy, x + dist * dx), 0.4 - 0.02 * (2 * i + j))]
    plant(vol[2], pairs)
    names[2] = "pairs 2 and 3 apart"
    corners = [(z, y, x) for z in (0, 63) for y in (0, 127) for x in (0, 127)]
    edges = [(z, y, 64) for z in (0, 63) for y in (0, 127)] + [(z, 64, x) for z in (0, 63) for x in (0, 127)] + \
            [(32, y, x) for y in (0, 127) for x in (0, 127)]
    faces = [(0, 64, 64), (63, 64, 64), (32, 0, 64), (32, 127, 64), (32, 64, 0), (32, 64, 127)]
    cells = corners + edges + faces
    plant(vol[3], [(c, 0.3 + 0.02 * i) for i, c in enumerate(cells)])
    names[3] = "faces, edges, corners"
    plant(vol[4], [((63, 40, 40), 0.9)])                                               # across a frame boundary in z
    plant(vol[5], [((0, 40, 40), 0.5)])
    names[4] = names[5] = "z = 63 over next frame's z = 0"
    plant(vol[6], [((20, 50, 127), 0.9), ((20, 51, 0), 0.5), ((30, 127, 64), 0.9), ((31, 0, 64), 0.5)])   # no wrap in x or y
    names[6] = "row / plane wrap"
    t = np.float32(THRESH)
    plant(vol[7], [((10, 10, 10), t), ((30, 30, 30), np.nextafter(t, np.float32(1))), ((50, 100, 100), 0.3)])
    names[7] = "at thresh / next above"
    names[8] = "empty"
    vol[9] = 0.5
    names[9] = "constant"
    vol[10] = synth.bev_noise_volume(21)[0]
    names[10] = "dense noise"
    vol[11] = dense_frame(22)
    names[11] = "dense noise + 80 peaks"
    vol[12] = tie_frame(23)
    names[12] = "dense ties"
    vol[13] = rs.uniform(0, 0.05, size=(64, 128, 128))                                # 65..4096 maxima: the sorted
    plant(vol[13], lattice_peaks(rs, 3000))                                            # candidate list, cut to 64
    names[13] = "3000 peaks"
    vol[14] = rs.uniform(0, 0.05, size=(64, 128, 128))
    plant(vol[14], lattice_peaks(rs, 300, levels=60))                                  # ~5 equal peaks per value
    names[14] = "300 peaks, ties"
    for b in range(15, 32):
        vol[b] = dense_frame(100 + b, n_peaks=64 + b)
        names[b] = "dense noise + peaks"
    return vol, names


@pytest.fixture(scope="module")
def edges():
    vol, names = edge_batch()
    return vol, names, run_parse(torch.from_numpy(vol).to(DEV))


def rows_of(res, b):
    bi, czyx, conf = res
    return czyx[bi == b], conf[bi == b]


def test_parse_edges_batch32(edges):
    vol, names, gpu = edges
    res = assert_parse_exact(vol, gpu=gpu)
    bi, czyx, conf = res
    assert np.bincount(bi, minlength=32).tolist() == [6, 4, 12, 26, 1, 1, 4, 2, 0] + [64] * 23
    z, _ = rows_of(res, 1)
    assert z.tolist() == [[10, 20, 30], [10, 20, 31], [40, 90, 7], [41, 90, 7]]       # ties: index order
    z, _ = rows_of(res, 2)                                                              # 2 apart (y = 10): only the larger
    assert sorted(c[1] for c in z.tolist()) == [10] * 4 + [40] * 4 + [40, 40, 43, 43]
    z, c = rows_of(res, 7)
    assert z.tolist() == [[50, 100, 100], [30, 30, 30]] and c[1] == np.nextafter(np.float32(THRESH), np.float32(1))
    z, _ = rows_of(res, 9)
    assert (z[:, 0] * 16384 + z[:, 1] * 128 + z[:, 2]).tolist() == list(range(64))
    for b in [11] + list(range(13, 32)):                                                # the planted peaks are the top-64
        z, c = rows_of(res, b)
        assert len(z) == 64 and (c >= 0.25).all()


@pytest.mark.parametrize("frame", [0, 3, 9, 10, 11, 12, 13, 14])
def test_parse_frame_alone_equals_in_batch(edges, frame):
    vol, names, gpu = edges
    bi, czyx, conf = assert_parse_exact(np.ascontiguousarray(vol[frame:frame + 1]))
    z, c = rows_of(gpu[1:], frame)
    assert np.array_equal(czyx, z) and np.array_equal(conf, c), names[frame]


def test_parse_dense_batch32():
    """Every frame has > 4096 local maxima above the threshold: the top-64 of each is still exact."""
    vol = np.stack([dense_frame(200 + b) if b % 2 else synth.bev_noise_volume(200 + b)[0] for b in range(32)])
    bi, _, _ = assert_parse_exact(vol)
    assert np.bincount(bi, minlength=32).tolist() == [64] * 32


def test_parse_capacity_and_thresh0(edges):
    vol, names, gpu = edges
    vol_dev = torch.from_numpy(vol).to(DEV)
    for cap in (100, 1000):                                                             # clamp: the first rows of the full parse
        k, bi, czyx, conf = run_parse(vol_dev, THRESH, cap)
        assert k == cap and np.array_equal(bi, gpu[1][:cap]) and np.array_equal(czyx, gpu[2][:cap])
    v = np.zeros((3, 64, 128, 128), np.float32)
    v[0] = -1.0                                                                         # negative maxima
    plant(v[0], [((5, 5, 5), -0.5), ((40, 60, 60), -0.25)])
    plant(v[1], [((7, 8, 9), 1e-40), ((30, 30, 30), 0.3)])                              # a subnormal maximum is > 0
    bi, czyx, _ = assert_parse_exact(v, 0.0)
    assert bi.tolist() == [1, 1] and czyx.tolist() == [[30, 30, 30], [7, 8, 9]]


# ================================================================================================ regress + unpack
def face_and_interior_rows(n_frames, seed):
    """every face / edge / corner class of z in {0,1,2,61,62,63}, y and x in FACE, then interior cells, over the frames."""
    zs = [0, 1, 2, 61, 62, 63]
    cells = [(z, y, x) for z in zs for y in FACE for x in FACE]
    rs = np.random.RandomState(seed)
    cells += [(rs.randint(3, 61), rs.randint(3, 125), rs.randint(3, 125)) for _ in range(40)]
    bi = np.arange(len(cells)) % n_frames
    return np.sort(bi, kind="stable"), np.array(cells, np.int64)


def check_regress(m, sd64, maps_fv, bv, fv, dtype, code, bi, czyx, cap=None, count=None, name=""):
    n_rows = len(bi)
    cap = cap or n_rows
    bi_d = torch.full((cap,), SENT, dtype=torch.int64, device=DEV)
    cz_d = torch.full((cap, 3), SENT, dtype=torch.int64, device=DEV)
    bi_d[:n_rows] = torch.as_tensor(bi, device=DEV)
    cz_d[:n_rows] = torch.as_tensor(czyx, device=DEV)
    n, o = run_regress(m, maps_fv, bv, fv, code, n_rows if count is None else count, bi_d, cz_d, cap)
    bi_t, cz_t = bi_d[:n], cz_d[:n]
    # cams: the full-volume fp64 refiner sampled at the detections
    cref = torch.zeros(n, 3, dtype=torch.float64, device=DEV)
    ccond = torch.zeros_like(cref)
    for b in sorted(set(bi_t.tolist())):
        r = (bi_t == b).nonzero()[:, 0]
        ref, cond = cam_volume_fp64(sd64, maps_fv[b], bv[b])
        z, y, x = cz_t[r, 0], cz_t[r, 1], cz_t[r, 2]
        cref[r], ccond[r] = ref[:, z, y, x].T, cond[:, z, y, x].T
    cams = o["pp"][:, :3]
    worst_cam = check_bound(f"cams {name}", cams, cref, ccond, G_CAM)
    # cam_czyx: bit-exact on the GPU's own fp32 cams.  Where fp64 picks another cell, the decision boundary between the
    # two (the midpoint of two neighbouring anchors for z, the integer edge of (c+1)/2*128 for y and x) lies within the
    # cam's bound of the fp32 cam
    anchors = torch.from_numpy(synth.bev_cam3dmap_anchor())
    a64, c32, c64 = anchors.double(), cams.cpu(), cref.cpu()
    cc = o["cc"].cpu()
    assert torch.equal(cc, B.cam_to_centermap_coords(c32.clone(), anchors))
    cc64 = B.cam_to_centermap_coords(c64.clone(), a64)
    k32 = torch.argmin((c32[:, :1] - anchors[None]).abs(), 1)
    k64 = torch.argmin((c64[:, :1] - a64[None]).abs(), 1)
    assert ((k32 - k64).abs() <= 1).all() and ((cc - cc64)[:, 1:].abs() <= 1).all()
    moved = torch.cat([(k32 != k64)[:, None], (cc != cc64)[:, 1:]], 1)
    edge = torch.cat([((a64[k32] + a64[k64]) / 2)[:, None], 2 * torch.maximum(cc, cc64)[:, 1:].double() / 128 - 1], 1)
    slack = (G_CAM * U * ccond).cpu() + 4 * U * (c32.double().abs() + a64.max())     # + fp32 rounding of the cell arithmetic
    assert ((c32.double() - edge).abs()[moved] <= slack[moved]).all()
    print(f"cam_czyx {name}: {int(moved.sum())} of {3 * n} cells differ from fp64's choice, each at a decision boundary")
    # MLP at the GPU's own cam_czyx, bound propagated through the three layers
    cc_d = o["cc"]
    f = fv[bi_t, cc_d[:, 1], cc_d[:, 2]].double()
    emb = sd64["position_embeddings.weight"][cc_d[:, 0]]
    h, c = f + emb, f.abs() + emb.abs()
    for i in (0, 3, 6):
        w, bb = sd64[f"transformer.{i}.weight"], sd64[f"transformer.{i}.bias"]
        h, c = h @ w.T + bb, c @ w.abs().T + bb.abs()
        if i < 6:
            h = torch.relu(h)
    worst_mlp = check_bound(f"mlp {name}", o["pp"][:, 3:], h, c, G_MLP)
    # unpack
    pp = o["pp"]
    assert torch.equal(bits(o["cam"]), bits(pp[:, :3].contiguous())) and torch.equal(bits(o["be"]), bits(pp[:, 135:].contiguous()))
    assert (bits(o["th"][:, 66:]) == 0).all()
    x6 = pp[:, 3:135].double().reshape(-1, 3, 2)
    aa = O.rot6d_to_aa(x6.reshape(-1, 6)).reshape(n, 22, 3)
    # Gram-Schmidt of the two 6-D columns amplifies rounding by |a1| |a2| / |a1 x a2| (1 / sin of their angle)
    a1, a2 = x6[..., 0], x6[..., 1]
    gs = (a1.norm(dim=-1) * a2.norm(dim=-1) / torch.cross(a1, a2, dim=-1).norm(dim=-1)).reshape(n, 22, 1)
    err = (o["th"][:, :66].double().reshape(n, 22, 3) - aa).abs()
    tol = 1e-5 * torch.clamp(gs / 10.0, min=1.0)
    print(f"thetas {name}: max|err| vs fp64 {err.max().item() if n else 0.0:.2e}, worst err/tol {(err / tol).max().item() if n else 0.0:.3f}, "
          f"{int((gs > 10).sum())} joints with 1/sin > 10")
    assert (err <= tol).all()
    p = pp.double()
    tan = float(np.tan(np.radians(30.0)))
    den = p[:, 0] * tan + 1e-3
    depth = 1.0 / den
    tr = torch.stack([p[:, 2] * depth * tan, p[:, 1] * depth * tan, depth], 1)
    kappa = 4 * U * (p[:, 0].abs() * tan + 1e-3) / den.abs()                            # relative error of the fp32 depth
    check_bound(f"cam_trans {name}", o["tr"], tr, ((kappa / U + 4) * tr.abs().T).T, 2.0)
    return o, worst_cam, worst_mlp


def test_regress_model_state(model_state, sd64):
    precision, m = model_state
    b = m.buf
    dtype, code = ACT[precision]
    bi, czyx = face_and_interior_rows(3, 1)
    check_regress(m, sd64, b["maps_fv"], b["bv_out"], b["fv_feats"], dtype, code, bi, czyx, name=f"model {precision}")


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_regress_crafted_extremes(sd, sd64, precision):
    """Cam offsets that drive every cam component past +-1 (the [1,127] clamp) and cam[0] past both ends of the anchors
    (anchor 0 lands on cell 1, anchor 63 on cell 63); rows past a device count below the capacity stay untouched."""
    m = model(sd, precision)
    dtype, code = ACT[precision]
    nf = 12
    maps_fv, bv, fv = crafted_maps(nf, 7, dtype)
    for k in range(nf):                                                                 # channel 1..3, +-30, +-300
        maps_fv[k, 1 + (k // 4)] += (30.0 if k % 2 else -30.0) * (10.0 if (k // 2) % 2 else 1.0)
    bi, czyx = face_and_interior_rows(nf, 2)
    o, _, _ = check_regress(m, sd64, maps_fv, bv, fv, dtype, code, bi, czyx, name=f"extremes {precision}")
    cc = o["cc"].cpu()
    assert {1, 63} <= set(cc[:, 0].tolist()) and {1, 127} <= set(cc[:, 1].tolist()) and {1, 127} <= set(cc[:, 2].tolist())
    check_regress(m, sd64, maps_fv, bv, fv, dtype, code, bi[:50], czyx[:50], cap=len(bi), count=37, name=f"count<cap {precision}")


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_regress_full_capacity(sd, sd64, precision):
    """parse -> regress on the device count at full capacity: 64 rows x 32 dense frames = 2,048 rows."""
    m = model(sd, precision)
    dtype, code = ACT[precision]
    vol = torch.from_numpy(np.stack([dense_frame(300 + b) for b in range(32)])).to(DEV)
    k, bi, czyx, _ = run_parse(vol, THRESH)
    assert k == 2048
    del vol
    maps_fv, bv, fv = crafted_maps(32, 9, dtype)
    check_regress(m, sd64, maps_fv, bv, fv, dtype, code, bi, czyx, name=f"full {precision}")
