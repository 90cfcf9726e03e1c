"""BEV oracle (oracle/bev_oracle.py) against fixtures produced by the reference's own bev/ code."""
import os

import numpy as np
import torch

from oracle import bev_oracle as B
from oracle import romp_oracle as O
from romp_b200 import synth


def g(golden_dir, name):
    return np.load(os.path.join(golden_dir, name))


def planted_volume(z):
    rs = np.random.RandomState(int(z["noise_seed"]))
    _ = rs.choice(64 * 128 * 128, size=4096, replace=False)        # replay the generator's stream
    vol = np.zeros((1, 64, 128, 128), np.float32) + rs.uniform(0, 0.05, size=(1, 64, 128, 128)).astype(np.float32)
    for zz, y, x, v in z["planted_cells"]:
        vol[0, int(zz), int(y), int(x)] = v
    return vol


def test_bev_maps_and_model(golden_dir):
    z, zp = g(golden_dir, "bev_maps_seed0.npz"), g(golden_dir, "bev_parse.npz")
    sd = synth.bev_state_dict(0)
    frames = synth.synthetic_frames(1, seed=0)
    out = B.bev_model(sd, frames, 0.08, center3d_override=planted_volume(zp))
    c3d_own = B.coarse2fine(O.to_torch_sd(sd), O.hrnet32_forward(O.to_torch_sd(sd), torch.from_numpy(frames).float()))[0]
    assert np.abs(c3d_own.reshape(-1)[z["vox"]].numpy() - z["center3d_at"]).max() < 2e-4
    assert np.abs(out["cam_maps_3d"].reshape(3, -1)[:, z["vox"]].numpy() - z["cam3d_at"]).max() < 5e-4
    assert np.abs(out["center_map"][0, 0].numpy() - z["center_fv"]).max() < 2e-4
    assert np.abs(out["front_view_features"][0, :, 5::17, 3::19].numpy() - z["fv_pix"]).max() < 5e-4
    # parse + sampling + MLP on the planted volume: integers bit-exact
    assert np.array_equal(out["pred_batch_ids"].numpy(), zp["batch_ids"])
    assert np.array_equal(out["pred_czyxs"].numpy(), zp["czyx"])
    assert np.array_equal(out["center_confs"].numpy(), zp["conf"])
    assert np.array_equal(out["cam_czyx"].numpy(), zp["cam_czyx"])
    assert np.abs(out["params_pred"].numpy() - zp["params_pred"]).max() < 1e-3
    pk = O.pack_params(torch.from_numpy(zp["params_pred"]), num_betas=11)
    assert np.abs(pk["smpl_thetas"].numpy() - zp["smpl_thetas"]).max() < 1e-6
    assert np.array_equal(pk["smpl_betas"].numpy(), zp["smpl_betas"])
    assert np.abs(B.cam_to_trans(pk["cam"]).numpy() - zp["cam_trans"]).max() < 1e-5


def test_parse_3d_dense_noise(golden_dir):
    """More than 4,096 local maxima in one frame: the oracle's top-64 (value desc, index asc) is the reference's own."""
    z = g(golden_dir, "bev_parse_dense.npz")
    vol = synth.bev_noise_volume(int(z["seed"]))
    bi, czyx, conf = B.parse_3d(vol, float(z["thresh"]))
    assert int(z["n_maxima"]) > 4096 and len(bi) == 64
    assert np.array_equal(bi.numpy(), z["batch_ids"])
    assert np.array_equal(czyx.numpy(), z["czyx"])
    assert np.array_equal(conf.numpy(), z["conf"])
    assert np.array_equal(conf.numpy(), vol[0][tuple(z["czyx"].T)])


def test_bev_post(golden_dir):
    z = g(golden_dir, "bev_post.npz")
    pack_a, pack_s = synth.smpl_pack(0, num_betas=11), synth.smpl_pack(1)
    v, j = B.smpla_forward(pack_a, pack_s, z["betas"], z["thetas"])
    assert np.abs(v[:, z["vsel"]].numpy() - z["verts_sel"]).max() < 5e-6
    assert np.abs(j.numpy() - z["joints"]).max() < 5e-6
    trans = B.cam_to_trans(z["cam"])
    assert np.abs(trans.numpy() - z["cam_trans"]).max() < 1e-5
    # the reference converts pj2d to original-image pixels IN PLACE (post_parser.py:129-136), so the "pj2d" its NMS
    # sees is pj2d_org; the golden stores that aliased tensor
    pj = O.to_org_image(B.perspective_project(j, trans), [0, 512, 0, 512, 512, 512])
    assert np.abs(pj.numpy() - z["pj2d"]).max() < 2e-2          # pixels
    k1 = B.suppress_redundant(pj, z["cam"], (512, 512), 20)
    assert k1 == z["kept_after_nms"].tolist() and len(k1) == 7     # the near-duplicate (3) and the shadowed (8) go
    k2 = [k1[i] for i in B.remove_outlier(trans[k1], torch.from_numpy(z["cam"])[k1], 1.6)]
    assert k2 == z["kept_after_outlier"].tolist()
