"""BEV long-image (crowd) mode on the CPU: the crop plan and the stage-wise restatement of the filters against fixtures
produced by the reference's own process_long_image loop (tests/golden/make_golden_bev_long.py)."""
import os

import numpy as np
import pytest
import torch

from oracle import bev_oracle as B
from romp_b200 import synth
from romp_b200.bev import long_image_crop_table, long_image_plan
from tests import bev_long_oracle as L


@pytest.fixture(scope="module")
def post(golden_dir):
    return np.load(os.path.join(golden_dir, "bev_long_post.npz"))


@pytest.mark.parametrize("plan", [long_image_plan, L.long_image_plan], ids=["romp_b200", "oracle"])
def test_plan_matches_reference(post, plan):
    z = post
    starts = np.concatenate([[0], np.cumsum(z["plan_counts"])])
    for i, (h, w) in enumerate(z["plan_sizes"].tolist()):
        pad, boxes, info = plan(h, w, 0.8)
        ref = z["plan_boxes"][starts[i]:starts[i + 1]]
        assert pad == z["plan_pad"][i]
        assert boxes.dtype == np.int32 and np.array_equal(boxes, ref), (h, w)
        assert np.array_equal(info, z["plan_info"][i])
    pad, boxes, info = plan(int(z["h"]), int(z["w"]), 0.8)
    assert pad == z["pad_length"] and np.array_equal(boxes, z["boxes"]) and np.array_equal(info, z["pad_info"])


def test_plan_quirks(post):
    """The narrow last crop, h+1-wide crops and the crop counts of the issue's examples."""
    assert len(long_image_plan(256, 512, 0.8)[1]) == 14
    _, b, _ = long_image_plan(1080, 3840, 0.8)
    assert len(b) == 22 and b[1].tolist() == [215, 1296, 0, 1080] and b[-1, 1] - b[-1, 0] == 911
    _, b, _ = long_image_plan(256, 512, 0.8)
    assert b[-1, 1] - b[-1, 0] == 206


def test_crop_table(post):
    z = post
    tab = long_image_crop_table(z["boxes"], int(z["pad_length"]), int(z["h"]), int(z["w"]), 20.0)
    k = len(z["boxes"])
    assert tab.shape == (k, 6) and tab.dtype == np.float32
    assert np.isinf(tab[-1, 0]) and np.isinf(tab[0, 1]) and np.isinf(tab[1, 1]) and np.isfinite(tab[2:, 1]).all()
    assert tab[0, 4] == np.float32(0.5) and tab[-1, 2] == 256


def crops_from(z, packs):
    k = len(z["boxes"])
    crops = []
    for c in range(k):
        sel = np.where(z["crop_of"] == c)[0]
        if len(sel) == 0:
            crops.append(None)
            continue
        v, j = B.smpla_forward(packs[0], packs[1], z["betas"][sel], z["thetas"][sel])
        crops.append({"cam": torch.from_numpy(z["cam"][sel]), "center_confs": torch.from_numpy(z["conf"][sel]),
                      "smpl_betas": torch.from_numpy(z["betas"][sel]), "smpl_thetas": torch.from_numpy(z["thetas"][sel]),
                      "params_pred": torch.from_numpy(z["params_pred"][sel]), "verts": v, "joints": j, "ids": sel})
    return crops


def test_oracle_stages_match_reference(post):
    z = post
    packs = (synth.smpl_pack(0, num_betas=11), synth.smpl_pack(1))
    crops = crops_from(z, packs)
    stages, out = L.long_image_post(crops, z["boxes"], int(z["pad_length"]), int(z["h"]), int(z["w"]))
    n = len(z["cam"])
    for key in ("boundary", "nms", "outlier"):
        alive = np.zeros(n, bool)
        for c, st in stages.items():
            if isinstance(c, int):
                alive[crops[c]["ids"][st[key]]] = True
        assert np.array_equal(alive, z["alive_" + key]), key
    ids = out["params_pred"][:, 145].round().long().numpy()
    assert ids.tolist() == z["final_ids"].tolist()
    assert len(z["merged_nms"]) > len(z["final_ids"]) and len(z["merged_in"]) > len(z["merged_nms"])
    assert np.array_equal(out["cam"].numpy(), z["out_cam"])                     # fp32 cam conversion: bit-exact
    assert np.array_equal(out["center_confs"].numpy(), z["out_conf"]) and np.array_equal(out["params_pred"].numpy(), z["out_params_pred"])
    assert np.array_equal(out["pred_batch_ids"].numpy(), z["out_batch_ids"])
    rel = lambda a, b: np.abs(a - b).max() / np.abs(b).max()
    assert rel(out["cam_trans"].numpy(), z["out_cam_trans"]) < 1e-5
    assert rel(out["pj2d_org"].numpy(), z["out_pj2d_org"]) < 1e-5
    assert np.abs(out["joints"].numpy() - z["out_joints"]).max() < 1e-4
    assert np.abs(out["verts"].numpy()[:, z["vsel"]] - z["out_verts_sel"]).max() < 1e-4


def test_all_empty_is_none(post):
    z = post
    stages, out = L.long_image_post([None] * len(z["boxes"]), z["boxes"], int(z["pad_length"]), int(z["h"]), int(z["w"]))
    assert out is None
