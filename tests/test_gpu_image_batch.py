"""Batched inference on raw images of mixed sizes: b200romp_preprocess_bgr_batch (one kernel for n images of different
sizes, with a device pad table), ROMP.forward_images / forward_image_batches against the one-image forward, BEV
forward_images against per-frame forward_batch, and per-frame geometry in projection and in BEV's duplicate suppression."""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch

from oracle import preproc_oracle as P
from oracle import romp_oracle as O
from romp_b200 import ROMP, _lib, romp_settings, synth
from romp_b200.bev import BEV, bev_settings
from romp_b200.main import padding_image

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
from make_golden_preproc import CASES_OPENCV, checksum, images  # noqa: E402

pytestmark = pytest.mark.gpu


def batch_preprocess(imgs, size=512):
    """b200romp_preprocess_bgr_batch on device tensors (any row stride) -> frames [n,size,size,3], pad table [n,6]."""
    ts = [torch.from_numpy(np.ascontiguousarray(x)).cuda() if isinstance(x, np.ndarray) else x for x in imgs]
    n = len(ts)
    out = torch.empty((n, size, size, 3), dtype=torch.uint8, device="cuda")
    pad = torch.full((n, 6), -1.0, device="cuda")
    ia = lambda v: (C.c_int * n)(*v)
    _lib.check(_lib.load().b200romp_preprocess_bgr_batch(
        (C.c_void_p * n)(*[t.data_ptr() for t in ts]), ia([t.shape[0] for t in ts]), ia([t.shape[1] for t in ts]),
        ia([t.stride(0) for t in ts]), n, size, C.c_void_p(out.data_ptr()), C.c_void_p(pad.data_ptr()),
        C.c_void_p(torch.cuda.current_stream().cuda_stream)), "preprocess_bgr_batch")
    torch.cuda.synchronize()
    return out.cpu().numpy(), pad.cpu().numpy()


def single_preprocess(img, size=512):
    d = torch.from_numpy(np.ascontiguousarray(img)).cuda()
    out = torch.empty((size, size, 3), dtype=torch.uint8, device="cuda")
    pad = (C.c_float * 6)()
    _lib.check(_lib.load().b200romp_preprocess_bgr(C.c_void_p(d.data_ptr()), img.shape[0], img.shape[1], 3 * img.shape[1], size,
                                                   C.c_void_p(out.data_ptr()), pad, C.c_void_p(torch.cuda.current_stream().cuda_stream)))
    torch.cuda.synchronize()
    return out.cpu().numpy(), np.array(list(pad), np.float32)


def odd_images():
    rs = np.random.RandomState(4)
    return [rs.randint(0, 256, (h, w, 3)).astype(np.uint8) for h, w in [(1, 1), (2, 301), (257, 255), (1080, 1920), (37, 53)]]


# ------------------------------------------------------------------------------------------------
# 1. batched preprocessing == the single-image entry, bit for bit
# ------------------------------------------------------------------------------------------------
def test_batch_preprocess_equals_single_and_golden():
    g = np.load(os.path.join(HERE, "golden", "preproc_opencv.npz"))
    gold = images(CASES_OPENCV)
    imgs = gold + odd_images()
    frames, pad = batch_preprocess(imgs)
    for i, img in enumerate(imgs):
        one, pad1 = single_preprocess(img)
        assert np.array_equal(frames[i], one), f"image {i} {img.shape}"
        assert np.array_equal(pad[i], pad1) and np.array_equal(pad[i], padding_image(img)[1]), f"pad info {i}"
        if i < len(gold):
            assert np.array_equal(pad[i], g[f"pad{i}"])
            if CASES_OPENCV[i][2] == 512:                  # the golden's 512 cases: sample + checksum
                assert np.array_equal(frames[i][None].reshape(-1)[::97], g[f"sample{i}"]), f"case {i}"
                assert np.array_equal(checksum(frames[i][None]), g[f"sum{i}"]), f"case {i}"
    rev, pad_rev = batch_preprocess(imgs[::-1])
    assert np.array_equal(rev, frames[::-1]) and np.array_equal(pad_rev, pad[::-1])


def test_batch_preprocess_strided_device_images_and_many_launches():
    rs = np.random.RandomState(8)
    base = torch.from_numpy(rs.randint(0, 256, (300, 500, 3)).astype(np.uint8)).cuda()
    views = [base[:97, 10:130], base[5:6, 3:4], base[20:290, 7:407], base]   # row stride 1500 bytes > 3w
    assert views[0].stride(0) == 1500 and not views[0].is_contiguous()
    frames, pad = batch_preprocess(views)
    for i, v in enumerate(views):
        one, pad1 = single_preprocess(v.cpu().numpy())
        assert np.array_equal(frames[i], one) and np.array_equal(pad[i], pad1), i
    # more images than one launch takes (64): the remaining ones go in a second launch, in order
    small = [rs.randint(0, 256, (rs.randint(1, 40), rs.randint(1, 40), 3)).astype(np.uint8) for _ in range(70)]
    frames, pad = batch_preprocess(small, size=32)
    for i, img in enumerate(small):
        xo, po = P.img_preprocess(img, 32)
        assert np.array_equal(frames[i], xo[0]) and np.array_equal(pad[i], po), i


# ------------------------------------------------------------------------------------------------
# 2./3. ROMP: forward_images == [forward(img) for img in images]; the streaming generator == forward_images
# ------------------------------------------------------------------------------------------------
def mixed_images(seed):
    rs = np.random.RandomState(seed)
    shapes = [(300, 400), (640, 480), (200, 260), (1080, 1920), (37, 53)]
    imgs = [rs.randint(0, 256, (h, w, 3)).astype(np.uint8) for h, w in shapes]
    imgs[2] = np.tile(np.array([0, 0, 255], np.uint8), (200, 260, 1))      # a flat red image: the lowest center peaks
    return imgs


@pytest.fixture(scope="module")
def romp_params():
    sd, pack = synth.romp_state_dict(0), synth.smpl_pack(0)
    frames = np.concatenate([P.img_preprocess(x, 512)[0] for x in mixed_images(7)])
    c, _ = O.romp_maps(sd, frames)
    sd2, _, _ = synth.calibrate_center_head(sd, c.numpy(), max_per_frame=6)
    return sd2, pack


def romp_model(params, precision, max_batch, extra=()):
    return ROMP(romp_settings(["--precision", precision, "--max_batch", str(max_batch), *extra]), state_dict=params[0],
                smpl_pack=params[1])


def leave_one_frame_empty(m, imgs):
    """Set the detection threshold between the lowest per-image top center peak (of this engine's own maps) and the next
    lowest: that image has nobody in it, every other image has at least one person.  Returns the empty image's index."""
    n = len(imgs)
    fd = torch.empty((n, 512, 512, 3), dtype=torch.uint8, device="cuda")
    for i, img in enumerate(imgs):
        fd[i] = torch.from_numpy(single_preprocess(img)[0]).cuda()
    tops = []
    for i in range(n):
        with torch.cuda.stream(m.stream):
            c, _ = m.run_maps(fd[i:i + 1])
        m.stream.synchronize()
        tops.append(float(synth.nms_peaks(c.cpu().numpy())[0][0].max()))
    order = np.argsort(tops)
    m.settings.center_thresh = 0.5 * (tops[order[0]] + tops[order[1]])
    assert m.settings.center_thresh >= 0
    return int(order[0])


def assert_same(a, b, where):
    assert (a is None) == (b is None), where
    if a is None:
        return
    assert set(a) == set(b), where
    for k in a:
        assert a[k].dtype == b[k].dtype and np.array_equal(a[k], b[k]), f"{where}: {k}"


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_romp_forward_images_equals_forward(romp_params, precision):
    imgs = mixed_images(7)
    m = romp_model(romp_params, precision, 2)
    empty = leave_one_frame_empty(m, imgs)
    ref = [m(img) for img in imgs]
    got = m.forward_images(imgs)
    assert len(got) == len(imgs)
    assert got[empty] is None and all(ref[i] is not None for i in range(len(imgs)) if i != empty)
    for i in range(len(imgs)):
        assert_same(got[i], ref[i], f"image {i} {imgs[i].shape}")
        if got[i] is not None:
            assert "pred_batch_ids" not in got[i]
    # device tensors in, the same results
    dev = m.forward_images([torch.from_numpy(x).cuda() for x in imgs])
    for i in range(len(imgs)):
        assert_same(dev[i], ref[i], f"device image {i}")


def test_romp_image_batches_stream_equals_forward_images(romp_params):
    m = romp_model(romp_params, "bf16", 2)
    lists = [mixed_images(7)[:3], mixed_images(8)[1:], mixed_images(9), [mixed_images(10)[3]]]
    lists[2] = [torch.from_numpy(x).cuda() for x in lists[2]]                    # one list of device-resident images
    lists[2][0] = torch.from_numpy(np.pad(mixed_images(9)[0], ((0, 0), (0, 7), (0, 0)))).cuda()[:, :400]   # row stride > 3w
    ref = [m.forward_images(li) for li in lists]
    got = list(m.forward_image_batches(iter(lists)))
    assert len(got) == len(ref)
    for j, (a, b) in enumerate(zip(got, ref)):
        assert len(a) == len(b) == len(lists[j])
        for i in range(len(a)):
            assert_same(a[i], b[i], f"list {j} image {i}")
    # consecutive lists really differ (a stale slot would repeat the previous results)
    first = lambda res: next(r for r in res if r is not None)
    assert sum(r is not None for li in got for r in li) >= 6
    for j in range(len(got) - 1):
        assert not np.array_equal(first(got[j])["smpl_thetas"], first(got[j + 1])["smpl_thetas"])
    assert list(m.forward_image_batches([[]])) == [[]]


def test_romp_temporal_is_not_batched(romp_params):
    m = romp_model(romp_params, "bf16", 2, ["--temporal_optimize"])
    with pytest.raises(NotImplementedError):
        m.forward_images(mixed_images(7)[:2])


# ------------------------------------------------------------------------------------------------
# 5. per-frame offsets in ROMP.forward_batch: each frame projects to its own image
# ------------------------------------------------------------------------------------------------
def test_romp_forward_batch_per_frame_offsets():
    sd, pack = synth.romp_state_dict(0), synth.smpl_pack(0)
    imgs = mixed_images(3)[:4]
    frames, pads = zip(*[P.img_preprocess(x, 512) for x in imgs])
    frames, pads = np.concatenate(frames), np.stack(pads)
    planted, _ = synth.plant_centers(4, seed=2)
    m = romp_model((sd, pack), "fp32", 4)
    out = m.forward_batch(torch.from_numpy(frames), offsets=pads, center_override=torch.from_numpy(planted).cuda())
    ids = out["pred_batch_ids"]
    assert sorted(set(ids.tolist())) == [0, 1, 2, 3]
    for b in range(4):
        r = ids == b
        pr = O.project_outputs(torch.from_numpy(out["joints"][r]), None, torch.from_numpy(out["cam"][r]), pads[b])
        err = np.abs(out["pj2d_org"][r] - pr["pj2d_org"].numpy()).max()
        print(f"frame {b} {imgs[b].shape}: pj2d_org max err {err:.2e} px")
        assert err < 0.02
    # the same frames with one shared pad info still take the old path
    one = m.forward_batch(torch.from_numpy(frames), offsets=pads[1], center_override=torch.from_numpy(planted).cuda())
    r = ids == 1
    assert np.array_equal(one["pj2d_org"][r], out["pj2d_org"][r])
    assert not np.array_equal(one["pj2d_org"][ids == 0], out["pj2d_org"][ids == 0])


# ------------------------------------------------------------------------------------------------
# 4. BEV forward_images: normal images of mixed sizes + one wide (crowd-mode) image
# ------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def bev_params():
    return synth.bev_damp_cam_offsets(synth.bev_state_dict(0)), synth.smpl_pack(0, num_betas=11), synth.smpl_pack(1)


def bev_volumes(n):
    """Planted 3-D centre maps.  Frame 0 (a 1080x1920 image) holds pairs of persons 3..6 cells apart: under its own
    max(h, w) some of them are duplicates, under 512 none is."""
    vol = np.random.RandomState(5).uniform(0, 0.05, size=(n, 64, 128, 128)).astype(np.float32)
    for k, (y, x, dx) in enumerate([(50, 20, 3), (50, 60, 4), (80, 20, 5), (80, 60, 6), (65, 100, 3)]):
        vol[0, 34, y, x] = 0.9 - 0.05 * k
        vol[0, 34, y, x + dx] = 0.85 - 0.05 * k
    for b in range(1, n):
        for k, (y, x) in enumerate([(40, 40), (40, 90), (90, 64)][:b + 1]):
            vol[b, 30 + 2 * k, y, x] = 0.8 - 0.1 * k
    return vol


def test_bev_forward_images(bev_params):
    s = bev_settings(["--precision", "fp32", "--max_batch", "2"])
    m = BEV(s, state_dict=bev_params[0], smpla_pack=bev_params[1], smil_pack=bev_params[2])
    rs = np.random.RandomState(21)
    normal = [rs.randint(0, 256, (h, w, 3)).astype(np.uint8) for h, w in [(1080, 1920), (480, 640), (1280, 720)]]
    wide = rs.randint(0, 256, (1080, 3840, 3)).astype(np.uint8)
    imgs = [normal[0], wide, normal[1], normal[2]]
    vol = torch.from_numpy(bev_volumes(3)).cuda()
    got = m.forward_images(imgs, center3d_override=vol)
    assert len(got) == 4
    differs = False
    for i, img in enumerate(normal):
        frame, pad = single_preprocess(img)
        side = float(max(img.shape[:2]))
        ref = m.forward_batch(torch.from_numpy(frame[None]), offsets=pad, img_max_side=side, center3d_override=vol[i:i + 1])
        assert ref is not None
        assert_same(got[[0, 2, 3][i]], ref, f"normal image {i} {img.shape}")
        at512 = m.forward_batch(torch.from_numpy(frame[None]), offsets=pad, img_max_side=512.0, center3d_override=vol[i:i + 1])
        if len(at512["cam"]) != len(ref["cam"]):
            differs = True
    assert differs, "no frame's duplicate suppression depends on its own size: the test lost its power"
    assert_same(got[1], m.process_long_image(wide), "wide image")
    # per-frame offsets in forward_batch: the batch of GPU frames with its pad table == forward_images
    frames = np.stack([single_preprocess(x)[0] for x in normal])
    pads = np.stack([padding_image(x)[1] for x in normal])
    m3 = BEV(bev_settings(["--precision", "fp32", "--max_batch", "3"]), state_dict=bev_params[0], smpla_pack=bev_params[1],
             smil_pack=bev_params[2])
    out = m3.forward_batch(torch.from_numpy(frames), offsets=pads, center3d_override=vol)
    for i in range(3):
        r = out["pred_batch_ids"] == i
        for k in ("cam", "verts", "pj2d_org", "center_confs"):
            assert np.array_equal(out[k][r], got[[0, 2, 3][i]][k]), (i, k)
