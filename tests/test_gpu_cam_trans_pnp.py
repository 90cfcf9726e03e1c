"""``--cam_trans epnp``: the reference's default cam_trans (estimate_translation, utils.py:391-436: validity mask, then
cv2.solvePnPRansac(EPnP, 20 px, 100 iterations)) as OpenCV's RANSAC loop around the published EPnP on the device
(csrc/pnp.cu), checked against the fp64 restatement in tests/pnp_oracle.py.

1. CPU: the restatement's RANSAC loop with cv2.solvePnP(EPNP) as its kernel against cv2.solvePnPRansac on a seeded
   population of SMPL people (outliers, joints above the image top, n from 24 down to 3): the same inlier set on every
   person, and the same tvec.  The gap of the published EPnP to OpenCV 4.13's is printed.
2. GPU: b200romp_cam_trans_pnp against the restatement with the published EPnP: inlier masks equal (a person where a joint
   came within 1e-3 px² of the 400 px² threshold is counted and printed), cam_trans within 1e-6 relative, INVALID rows,
   the device count, and bit-identical results at 1, 7 and 640 persons.
3. GPU, whole path: forward_batch with --cam_trans epnp against lsq and the restatement; forward_batches, forward_images
   and forward_video (tracked and --show_largest) against their per-frame forward loops."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import romp_oracle as O
from romp_b200 import synth
from tests import pnp_oracle as PO

N_POP = 2048


def population(n=N_POP, seed=0):
    """SMPL joints [n,71,3] (oracle forward on synth.smpl_pack, random poses and shapes) and cams [n,3] with the scale
    log-uniform in [0.2, 4] and the shift in [-0.6, 0.6].  A quarter of the people get 1-8 joints moved in depth (outliers
    under perspective); a quarter have the k topmost joints pushed above the image top (k in 0..21, so n = 24..3, with
    n = 5, 4 and 3 each forced on a few); a few have joints with z = -2."""
    rs = np.random.RandomState(seed + 31337)
    pack = synth.smpl_pack(0)
    thetas = rs.normal(0, 0.35, (n, 72)).astype(np.float32)
    thetas[:, :3] = rs.normal(0, 1.0, (n, 3))
    betas = rs.normal(0, 1.0, (n, 10)).astype(np.float32)
    joints = np.concatenate([O.smpl_forward(pack, betas[i:i + 256], thetas[i:i + 256])[1].numpy() for i in range(0, n, 256)])
    cam = np.stack([np.exp(rs.uniform(np.log(0.2), np.log(4.0), n)), rs.uniform(-0.6, 0.6, n), rs.uniform(-0.6, 0.6, n)],
                   1).astype(np.float32)
    kind = rs.randint(0, 4, n)
    for i in np.flatnonzero(kind == 1):
        idx = rs.choice(24, rs.randint(1, 9), replace=False)
        joints[i, idx, 2] += rs.choice([-1, 1], len(idx)) * rs.uniform(0.3, 1.5, len(idx)).astype(np.float32)
    for j, i in enumerate(np.flatnonzero(kind == 2)):
        k = [19, 20, 21][j] if j < 3 else (19 + j % 3 if j < 24 else rs.randint(0, 22))
        ys = np.sort(joints[i, :24, 1] * cam[i, 0])
        lo = ys[k - 1] if k > 0 else ys[0] - 0.05
        cam[i, 2] = np.float32(-1.0 - 2.0 / 256.0 - 0.5 * (lo + ys[k]))
    for i in np.flatnonzero(kind == 3)[:40]:
        joints[i, rs.choice(24, 2, replace=False), 2] = -2.0
    return joints.astype(np.float32), cam


@pytest.fixture(scope="module")
def pop():
    return population()


def valid_counts(joints, cam):
    return PO.pj2d_valid(joints, cam)[2].sum(1)


def cv2_ransac(joints, cam):
    """cv2.solvePnPRansac per person on the valid joints, like estimate_translation (utils.py:412-431)."""
    import cv2
    j3, p2, valid = PO.pj2d_valid(joints, cam)
    out, bits = np.zeros((len(j3), 3)), np.zeros(len(j3), np.int64)
    for i in range(len(j3)):
        v = valid[i]
        if v.sum() < 4:
            out[i] = -1
            continue
        _, _, tvec, inl = cv2.solvePnPRansac(j3[i][v], p2[i][v], PO.K, None, flags=cv2.SOLVEPNP_EPNP, reprojectionError=20,
                                             iterationsCount=100)
        out[i] = -1 if inl is None else tvec[:, 0]
        bits[i] = 0 if inl is None else int(sum(1 << int(k) for k in inl.ravel()))
    return out, bits


# ------------------------------------------------------------------------------------------------
# 1. CPU: the RANSAC loop against cv2.solvePnPRansac
# ------------------------------------------------------------------------------------------------
def test_population_covers_the_cases(pop):
    n = valid_counts(*pop)
    assert (n == 24).sum() > 500 and (n < 4).sum() >= 3 and (n == 4).sum() >= 3 and (n == 5).sum() >= 3
    assert len(set(n.tolist())) >= 20, sorted(set(n.tolist()))


def test_ransac_loop_equals_cv2_solvePnPRansac(pop):
    pytest.importorskip("cv2")
    joints, cam = pop
    n = valid_counts(joints, cam)
    t_cv, bits_cv = cv2_ransac(joints, cam)
    t_re, bits_re, _ = PO.cam_trans_epnp(joints, cam, kernel="cv2")
    keep = n != 4                       # cv2 runs P3P on 4 points (out of scope)
    full = np.array([(1 << int(k)) - 1 for k in n])
    outliers = int(((bits_cv != full) & keep & (n >= 6)).sum())
    assert outliers >= 100, outliers
    assert np.array_equal(bits_re[keep], bits_cv[keep]), np.flatnonzero((bits_re != bits_cv) & keep)[:10]
    scale = np.maximum(np.abs(t_cv).max(1, keepdims=True), 1e-30)
    assert np.all(np.abs(t_re[keep] - t_cv[keep]) <= 1e-6 * scale[keep] + 1e-7), np.abs(t_re - t_cv)[keep].max()
    # cv2 on 4 points: P3P; where it succeeds every point is an inlier
    assert np.all((bits_cv[n == 4] == 0) | (bits_cv[n == 4] == 15))
    # the published EPnP as the kernel: how far it lands from OpenCV 4.13's
    t_ep, bits_ep, _ = PO.cam_trans_epnp(joints, cam)
    agree = keep & (bits_ep == bits_cv) & (t_cv[:, 2] != -1)
    big = agree & (n >= 6)
    rel = np.abs(t_ep[big] - t_cv[big]).max(1) / np.abs(t_cv[big]).max(1)
    print(f"\n{outliers} people with outliers; published EPnP vs cv2: inlier sets equal on "
          f"{int((bits_ep[keep] == bits_cv[keep]).sum())}/{int(keep.sum())}; on those with >= 6 points, cam_trans (float32) "
          f"relative gap median {np.median(rel):.1e}, max {rel.max():.1e}")
    assert (bits_ep[keep] == bits_cv[keep]).mean() > 0.9 and rel.max() < 1e-6


def test_subsets_follow_opencv_rng():
    s = PO.cv_rng_subsets(24)
    assert s.shape == (100, 5) and all(len(set(r)) == 5 for r in s.tolist())
    assert PO.ransac_update_num_iters(0.99, 0.0, 5, 100) == 0
    assert PO.ransac_update_num_iters(0.99, 0.5, 5, 100) == 100
    assert PO.ransac_update_num_iters(0.99, 0.2, 5, 100) == int(np.rint(np.log(0.01) / np.log(1 - 0.8 ** 5))) == 12


# ------------------------------------------------------------------------------------------------
# 2. GPU: the kernel against the restatement
# ------------------------------------------------------------------------------------------------
def run_device(joints, cam, count=None, fill=0.0):
    from romp_b200 import _lib
    lib = _lib.load()
    j, c = torch.from_numpy(joints).cuda(), torch.from_numpy(cam).cuda()
    out = torch.full((len(joints), 3), fill, dtype=torch.float32, device="cuda")
    mask = torch.full((len(joints),), -7, dtype=torch.int32, device="cuda")
    d = None if count is None else torch.tensor([count], dtype=torch.int32, device="cuda")
    p = lambda t: None if t is None else C.c_void_p(t.data_ptr())
    _lib.check(lib.b200romp_cam_trans_pnp(p(j), p(c), len(joints), p(d), p(out), p(mask),
                                          C.c_void_p(torch.cuda.current_stream().cuda_stream)), "cam_trans_pnp")
    torch.cuda.synchronize()
    return out.cpu().numpy(), mask.cpu().numpy().astype(np.int64) & 0xFFFFFFFF


@pytest.fixture(scope="module")
def restated(pop):
    return PO.cam_trans_epnp(*pop)


@pytest.mark.gpu
def test_kernel_equals_restatement(pop, restated):
    joints, cam = pop
    t_re, bits_re, near = restated
    t_dev, bits_dev = run_device(joints, cam)
    diff = np.flatnonzero(bits_dev != bits_re)
    ties = [i for i in diff if near[i] < 1e-3]
    for i in ties:
        print(f"person {i}: a joint {near[i]:.1e} px² from the threshold; masks {bits_dev[i]:#x} / {bits_re[i]:#x}")
    print(f"\n{len(ties)} people decided within 1e-3 px² of the threshold, {len(diff)} mask differences")
    assert set(diff.tolist()) == set(ties), [(i, near[i]) for i in diff if i not in ties][:10]
    same = np.setdiff1d(np.arange(len(joints)), diff)
    scale = np.abs(t_re[same]).max(1, keepdims=True)
    err = np.abs(t_dev[same] - t_re[same]) / scale
    print(f"max relative |device - restatement| cam_trans {err.max():.1e}")
    assert err.max() <= 1e-6
    inv = valid_counts(joints, cam) < 4
    assert inv.sum() >= 3 and np.all(t_dev[inv] == -1.0) and np.all(bits_dev[inv] == 0)


@pytest.mark.gpu
def test_kernel_device_count_and_person_counts(pop):
    joints, cam = pop
    full, bits = run_device(joints[:640], cam[:640])
    for m in (1, 7):
        t, b = run_device(joints[:m], cam[:m])
        assert np.array_equal(t.view(np.uint32), full[:m].view(np.uint32)) and np.array_equal(b, bits[:m])
    t, b = run_device(joints[:9], cam[:9], count=5, fill=7.0)
    assert np.array_equal(t[:5].view(np.uint32), full[:5].view(np.uint32)) and np.array_equal(b[:5], bits[:5])
    assert np.all(t[5:] == 7.0) and np.all(b[5:] == (-7 & 0xFFFFFFFF))
    t, _ = run_device(joints[:9], cam[:9], count=0, fill=7.0)
    assert np.all(t == 7.0)


# ------------------------------------------------------------------------------------------------
# 3. GPU, whole path
# ------------------------------------------------------------------------------------------------
def make(mode, max_batch=4, extra=()):
    from romp_b200 import ROMP, romp_settings
    sd, pack = _params()
    flags = ["--precision", "fp32", "--max_batch", str(max_batch), "--cam_trans", mode] + list(extra)
    return ROMP(romp_settings(flags), state_dict=sd, smpl_pack=pack)


_PARAMS = {}


def _params():
    """Synthetic weights with the centre head calibrated to a few people per image (as in test_gpu_romp_video)."""
    if not _PARAMS:
        from oracle import preproc_oracle as P
        sd = synth.romp_state_dict(0)
        c, _ = O.romp_maps(sd, np.concatenate([P.img_preprocess(x, 512)[0] for x in images_of(5)]))
        _PARAMS["p"] = (synth.calibrate_center_head(sd, c.numpy(), max_per_frame=6)[0], synth.smpl_pack(0))
    return _PARAMS["p"]


def planted(B, seed=3):
    maps, _ = synth.plant_centers(B, seed=seed, kmin=3, kmax=9)
    return torch.from_numpy(maps).cuda()


def frames_of(B, seed=5):
    return synth.synthetic_frames(B, seed=seed)


def images_of(B, seed=8):
    """A scene with small changes from image to image, in a few sizes."""
    rs = np.random.RandomState(seed)
    base = np.random.RandomState(0).randint(0, 256, (720, 720, 3)).astype(np.int16)
    shapes = [(480, 640), (512, 512), (300, 700), (720, 400)]
    return [np.ascontiguousarray(np.clip(base + rs.randint(-5, 6, base.shape), 0, 255).astype(np.uint8)[:h, :w])
            for h, w in (shapes[i % 4] for i in range(B))]


def same(a, b, where):
    assert (a is None) == (b is None), where
    if a is None:
        return
    assert set(a) == set(b), (where, set(a) ^ set(b))
    for k in a:
        assert np.array_equal(np.asarray(a[k]), np.asarray(b[k])), (where, k)


@pytest.mark.gpu
def test_forward_batch_epnp_against_lsq_and_restatement():
    B = 4
    frames, co = frames_of(B), planted(B)
    got = make("epnp").forward_batch(frames, center_override=co)
    ref = make("lsq").forward_batch(frames, center_override=co)
    assert set(got) == set(ref)
    for k in ref:
        if k != "cam_trans":
            assert np.array_equal(got[k], ref[k]), k
    t_re, bits, near = PO.cam_trans_epnp(got["joints"], got["cam"])
    tie = near < 1e-3
    scale = np.abs(t_re).max(1, keepdims=True)
    assert np.all((np.abs(got["cam_trans"] - t_re) <= 1e-6 * scale) | tie[:, None])
    n_valid = valid_counts(got["joints"], got["cam"])
    print(f"\n{len(n_valid)} people, valid joints {sorted(set(n_valid.tolist()))}, {int(tie.sum())} near-threshold")
    assert not np.array_equal(got["cam_trans"], ref["cam_trans"])


@pytest.mark.gpu
def test_mask_on_people_above_the_image_top():
    """A centre on the top row puts people partly above the frame: fewer than 24 valid joints reach the kernel."""
    B = 2
    maps = np.zeros((B, 1, 64, 64), np.float32)
    maps[0, 0, 0, 10], maps[0, 0, 0, 40], maps[0, 0, 30, 30] = 0.9, 0.8, 0.7
    maps[1, 0, 1, 20], maps[1, 0, 2, 50] = 0.9, 0.6
    co = torch.from_numpy(maps).cuda()
    m = make("epnp")
    got = m.forward_batch(frames_of(B, seed=9), center_override=co)
    t_re, _, near = PO.cam_trans_epnp(got["joints"], got["cam"])
    n_valid = valid_counts(got["joints"], got["cam"])
    print(f"\nvalid joints per person {n_valid.tolist()}")
    scale = np.abs(t_re).max(1, keepdims=True)
    assert np.all((np.abs(got["cam_trans"] - t_re) <= 1e-6 * scale) | (near < 1e-3)[:, None])
    # the same people with their cams shifted up past the image top
    cam = got["cam"].copy()
    cam[:, 2] -= 1.0
    t_dev, _ = run_device(np.ascontiguousarray(got["joints"]), cam)
    t_re2, _, near2 = PO.cam_trans_epnp(got["joints"], cam)
    n2 = valid_counts(got["joints"], cam)
    assert (n2 < 24).any(), n2
    ok = (np.abs(t_dev - t_re2) <= 1e-6 * np.abs(t_re2).max(1, keepdims=True)) | (near2 < 1e-3)[:, None]
    assert np.all(ok), n2


@pytest.mark.gpu
def test_entry_points_equal_forward_loop():
    imgs = images_of(6)
    co = planted(6, seed=11)
    m = make("epnp")
    loop = [m.forward_images([img], center_override=co[i:i + 1])[0] for i, img in enumerate(imgs)]
    fwd = m.forward(imgs[0])
    batch = m.forward_images(imgs, center_override=co)
    for i in range(len(imgs)):
        same(batch[i], loop[i], f"forward_images {i}")
    assert any(r is not None for r in loop)
    # forward() on the image's own centre map is forward_images of one image
    same(fwd, m.forward_images([imgs[0]])[0], "forward")
    # forward_batches against forward_batch per batch
    frames = frames_of(6, seed=2)
    parts = list(m.forward_batches([frames[:3], frames[3:]], center_override=co[:3]))
    for j, fr in enumerate([frames[:3], frames[3:]]):
        one = m.forward_batch(fr, center_override=co[:3])
        same(None if parts[j] is None else {k: np.array(v) for k, v in parts[j].items()}, one, f"forward_batches {j}")


@pytest.mark.gpu
@pytest.mark.parametrize("largest", [False, True])
def test_forward_video_equals_forward_loop(largest):
    imgs = images_of(7, seed=21)
    co = planted(7, seed=13)
    extra = ["-t"] + (["--show_largest"] if largest else [])
    ref_m = make("epnp", extra=extra)
    ref = []
    for i, img in enumerate(imgs):
        ref.append(ref_m.forward(img))
    got = make("epnp", extra=extra).forward_video(imgs)
    lsq = make("lsq", extra=extra).forward_video(imgs)
    n_people = 0
    for i in range(len(imgs)):
        assert (got[i] is None) == (ref[i] is None), i
        if ref[i] is None:
            continue
        n_people += len(ref[i]["cam"])
        for k in ref[i]:
            e = float(np.abs(np.asarray(got[i][k], np.float64) - ref[i][k]).max()) if np.asarray(ref[i][k]).size else 0.0
            assert e <= (1e-3 if k == "pj2d_org" else 1e-5 if k in ("verts", "joints", "cam_trans") else 1e-6), (i, k, e)
        t_re, _, near = PO.cam_trans_epnp(got[i]["joints"], got[i]["cam"])
        ok = (np.abs(got[i]["cam_trans"] - t_re) <= 1e-6 * np.abs(t_re).max(1, keepdims=True)) | (near < 1e-3)[:, None]
        assert np.all(ok), i
        assert np.array_equal(got[i]["smpl_thetas"], lsq[i]["smpl_thetas"])
    assert n_people > 0
