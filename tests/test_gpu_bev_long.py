"""BEV long-image (crowd) mode on the GPU: crop frames, the two new filter stages and the whole path against the
reference's own process_long_image loop (tests/golden/bev_long_*.npz) and the CPU restatement (tests/bev_long_oracle.py)."""
import os

import numpy as np
import pytest
import torch

from oracle import bev_oracle as B
from oracle import preproc_oracle as PO
from oracle import romp_oracle as O
from romp_b200 import synth
from romp_b200.bev import BEV, bev_settings, long_image_crop_table, long_image_plan
from romp_b200.main import img_preprocess
from tests import bev_long_oracle as L

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def params():
    return synth.bev_damp_cam_offsets(synth.bev_state_dict(0)), synth.smpl_pack(0, num_betas=11), synth.smpl_pack(1)


def make(params, precision, max_batch, extra=()):
    s = bev_settings(["--precision", precision, "--max_batch", str(max_batch), *extra])
    return BEV(s, state_dict=params[0], smpla_pack=params[1], smil_pack=params[2])


@pytest.fixture(scope="module")
def m16(params):
    return make(params, "fp32", 16)


def model_inputs(golden_dir):
    z = np.load(os.path.join(golden_dir, "bev_long_model.npz"))
    h, w = int(z["h"]), int(z["w"])
    image = L.long_image(h, w, int(z["image_seed"]))
    vols = L.planted_volumes(len(long_image_plan(h, w, 0.8)[1]), int(z["vol_seed"]))
    return z, image, vols


def test_crop_frames_bit_exact(m16):
    """Device crops of a 1080x3840 image == img_preprocess of the same boxes (OpenCV's own bicubic, IPP off)."""
    h, w = 1080, 3840
    image = L.long_image(h, w, 3)
    pad, boxes, _ = long_image_plan(h, w, 0.8)
    assert len(boxes) == 22
    pick = [0, 1, len(boxes) - 1]            # zero-padded left crop, an h+1-wide crop, the narrow last crop
    assert boxes[1, 1] - boxes[1, 0] == h + 1 and boxes[-1, 1] - boxes[-1, 0] == 911
    frames = torch.empty((len(pick), 512, 512, 3), dtype=torch.uint8, device="cuda")
    with torch.cuda.stream(m16.stream):
        padded = m16.pad_long_image(torch.from_numpy(image), pad)
        m16.crop_frames(padded, boxes[pick], frames)
    m16.stream.synchronize()
    host = np.zeros((h, w + 2 * pad, 3), np.uint8)
    host[:, pad:pad + w] = image
    assert np.array_equal(padded.cpu().numpy(), host)
    for i, k in enumerate(pick):
        l, r, t, b = boxes[k]
        ref, _ = PO.img_preprocess(host[t:b, l:r])
        assert np.array_equal(frames[i].cpu().numpy(), ref[0]), k


def test_stages_vs_reference(m16, golden_dir):
    """The per-crop and merged stages on the fixture's synthetic per-crop records."""
    z = np.load(os.path.join(golden_dir, "bev_long_post.npz"))
    m = m16
    h, w, pad, boxes = int(z["h"]), int(z["w"]), int(z["pad_length"]), z["boxes"]
    k = len(boxes)
    order = np.argsort(z["crop_of"], kind="stable")           # rows grouped by crop, like bev_parse3d leaves them
    n = len(order)
    b = m.buf
    put = lambda key, v: b[key][:n].copy_(torch.from_numpy(np.ascontiguousarray(v)).cuda())
    put("betas", z["betas"][order]); put("thetas", z["thetas"][order]); put("cam", z["cam"][order])
    put("cam_trans", B.cam_to_trans(torch.from_numpy(z["cam"][order])).numpy()); put("conf", z["conf"][order])
    put("params_pred", z["params_pred"][order]); put("batch_ids", z["crop_of"][order])
    b["count"][0] = n
    m._long_buffers(k * 64)
    tab = torch.from_numpy(long_image_crop_table(boxes, pad, h, w, 20.0)).cuda()
    torch.cuda.synchronize()
    with torch.cuda.stream(m.stream):
        m._long["count"].zero_()
        m.crop_post(k, 0, tab)
        m.long_merge(z["pad_info"], w)
    out = m._collect_long()
    lb = m._long
    n_acc = int(lb["count"][0])
    acc_ids = lb["params_pred"][:n_acc, 145].round().long().cpu().numpy()
    assert acc_ids.tolist() == z["merged_in"].tolist()                         # per-crop survivors, in crop order
    ids = out["params_pred"][:, 145].round().astype(np.int64)
    assert ids.tolist() == z["final_ids"].tolist()
    assert np.array_equal(out["cam"], z["out_cam"])                           # cam conversion bit-exact
    assert np.array_equal(out["center_confs"], z["out_conf"]) and np.array_equal(out["params_pred"], z["out_params_pred"])
    assert np.array_equal(out["smpl_thetas"], z["out_thetas"]) and np.array_equal(out["smpl_betas"], z["out_betas"])
    assert np.abs(out["verts"][:, z["vsel"]] - z["out_verts_sel"]).max() < 1e-4
    assert np.abs(out["joints"] - z["out_joints"]).max() < 1e-4
    assert np.abs(out["pj2d_org"] - z["out_pj2d_org"]).max() < 5e-2
    assert np.abs(out["cam_trans"] - z["out_cam_trans"]).max() < 1e-4 * np.abs(z["out_cam_trans"]).max()
    assert np.array_equal(out["pred_batch_ids"], np.zeros(len(ids), np.int64))


def test_end_to_end_fp32(m16, golden_dir):
    z, image, vols = model_inputs(golden_dir)
    out = m16.process_long_image(image, center3d_override=torch.from_numpy(vols).cuda())
    assert set(out) == {"smpl_thetas", "smpl_betas", "cam", "cam_trans", "params_pred", "center_confs", "pred_batch_ids",
                        "verts", "joints", "pj2d_org"}
    assert set(out) <= set(z["keys"].tolist())
    assert out["center_confs"].tolist() == z["center_confs"].tolist()            # the same survivors in the same order
    assert np.array_equal(out["pred_batch_ids"], np.zeros(len(out["cam"]), np.int64))
    print("cam err", np.abs(out["cam"] - z["cam"]).max(), "verts err", np.abs(out["verts"][:, z["vsel"]] - z["verts_sel"]).max())
    assert np.abs(out["cam"] - z["cam"]).max() < 2e-3
    assert np.abs(out["verts"][:, z["vsel"]] - z["verts_sel"]).max() < 2e-2
    assert np.abs(out["joints"] - z["joints"]).max() < 2e-2


def test_bf16_stagewise(params, golden_dir):
    """bf16 model: the oracle's steps 3-7 on the GPU's own per-crop params_pred give the same survivors and meshes."""
    z, image, vols = model_inputs(golden_dir)
    m = make(params, "bf16", 16)
    h, w = image.shape[:2]
    pad, boxes, _ = long_image_plan(h, w, 0.8)
    out = m.process_long_image(image, center3d_override=torch.from_numpy(vols).cuda())
    b = m.buf
    n = int(b["count"].item())
    pp = b["params_pred"][:n].cpu()
    bids = b["batch_ids"][:n].cpu().numpy()
    conf = b["conf"][:n].cpu()
    pk = O.pack_params(pp, num_betas=11)
    crops = []
    for c in range(len(boxes)):
        sel = np.where(bids == c)[0].tolist()
        if not sel:
            crops.append(None)
            continue
        v, j = B.smpla_forward(params[1], params[2], pk["smpl_betas"][sel], pk["smpl_thetas"][sel])
        crops.append({"cam": pk["cam"][sel], "center_confs": conf[sel], "smpl_betas": pk["smpl_betas"][sel],
                      "smpl_thetas": pk["smpl_thetas"][sel], "params_pred": pp[sel], "verts": v, "joints": j})
    _, ref = L.long_image_post(crops, boxes, pad, h, w)
    assert out["center_confs"].tolist() == ref["center_confs"].tolist()
    assert np.array_equal(out["cam"], ref["cam"].numpy())
    assert np.abs(out["verts"] - ref["verts"].numpy()).max() < 1e-4 and np.abs(out["joints"] - ref["joints"].numpy()).max() < 1e-4


def test_chunking_bit_equal(params, m16, golden_dir):
    _, image, vols = model_inputs(golden_dir)
    v = torch.from_numpy(vols).cuda()
    a = make(params, "fp32", 4).process_long_image(image, center3d_override=v)
    b = m16.process_long_image(image, center3d_override=v)
    assert set(a) == set(b)
    for key in a:
        assert np.array_equal(a[key], b[key]), key


def test_dispatch(params, m16, golden_dir):
    _, image, vols = model_inputs(golden_dir)
    assert image.shape[1] == 2 * image.shape[0]
    calls = []
    orig = m16.process_long_image
    m16.process_long_image = lambda img, **kw: calls.append(img.shape) or orig(img, center3d_override=torch.zeros(14, 64, 128, 128).cuda())
    try:
        assert m16(image) is None                 # exactly 2:1 takes the long path; nobody in any crop -> None
    finally:
        del m16.process_long_image
    assert calls == [image.shape]
    # --crowd (crowd off): the normal path, i.e. forward_batch on the host-padded 512x512 frame
    m = make(params, "fp32", 2, ["--crowd"])
    wide = L.long_image(200, 700, 9)
    out = m(wide)
    inp, pad = img_preprocess(wide)
    ref = m.forward_batch(torch.from_numpy(inp), offsets=pad, img_max_side=700.0)
    assert (out is None) == (ref is None)
    if out is not None:
        for key in out:
            assert np.array_equal(out[key], ref[key]), key
    m2 = make(params, "fp32", 2, ["--show_patch_results"])
    with pytest.raises(NotImplementedError):
        m2(image)
    m3 = make(params, "fp32", 2, ["--calc_smpl"])
    with pytest.raises(ValueError):
        m3(image)
