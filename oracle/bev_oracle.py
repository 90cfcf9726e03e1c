"""CPU oracle for the BEV variant of the hot path (workload cfg3).  TEST INFRASTRUCTURE ONLY.

fp32 torch-CPU restatement of simple_romp/bev/model.py (BEVv1.forward :232-250 and helpers) and
simple_romp/bev/post_parser.py (CenterMap3D.parse_3dcentermap :44-66, pack_params_dict :240-253,
denormalize_cam_params_to_trans :114-128, perspective_projection :68-107, SMPLA_parser :255-278,
suppressing_redundant_prediction_via_projection :167-198, remove_outlier :200-222).
Pinned by fixtures generated from the reference's own code (tests/golden/make_golden_bev.py).
"""
from __future__ import annotations

import math

import numpy as np
import torch
import torch.nn.functional as F

from . import romp_oracle as R

_t = R._t
TAN_FOV = float(np.tan(np.radians(60 / 2.0)))          # bev/post_parser.py:109


def _bn(sd, p, x):
    return F.batch_norm(x, sd[p + ".running_mean"], sd[p + ".running_var"], sd[p + ".weight"], sd[p + ".bias"],
                        False, 0.0, R.BN_EPS)


def head_block(sd, p, x):
    """BasicBlock(32->128) with a biased 1x1 downsample and no BN on it (bev/model.py:154-156, romp/model.py:67-83)."""
    y = F.relu(_bn(sd, p + "bn1", F.conv2d(x, sd[p + "conv1.weight"], None, 1, 1)))
    y = _bn(sd, p + "bn2", F.conv2d(y, sd[p + "conv2.weight"], None, 1, 1))
    res = F.conv2d(x, sd[p + "downsample.weight"], sd[p + "downsample.bias"])
    return F.relu(y + res)


def block_1d(sd, p, x):
    """BasicBlock_1D, bev/model.py:24-45 (no residual)."""
    y = F.relu(_bn(sd, p + "bn1", F.conv1d(x, sd[p + "conv1.weight"], None, 1, 1)))
    return F.relu(_bn(sd, p + "bn2", F.conv1d(y, sd[p + "conv2.weight"], None, 1, 1)))


def block_3d(sd, p, x):
    """BasicBlock_3D, bev/model.py:52-75 (residual, no final ReLU)."""
    y = F.relu(_bn(sd, p + "bn1", F.conv3d(x, sd[p + "conv1.weight"], None, 1, 1)))
    y = _bn(sd, p + "bn2", F.conv3d(y, sd[p + "conv2.weight"], None, 1, 1))
    return y + x


def fv_maps(sd, feat):
    """det_head and bv_pre_layers on the backbone features (bev/model.py:188-190) -> (maps_fv [B,4,128,128] = center_fv |
    cam_offset, img_feats [B,16,128,128])."""
    maps_fv = F.conv2d(head_block(sd, "det_head.0.0.", feat), sd["det_head.1.weight"], sd["det_head.1.bias"])
    x = feat
    for i in (0, 3, 6):
        w = sd[f"bv_pre_layers.{i}.weight"]
        x = F.relu(_bn(sd, f"bv_pre_layers.{i + 1}", F.conv2d(x, w, sd[f"bv_pre_layers.{i}.bias"], 1, w.shape[-1] // 2)))
    return maps_fv, x


def bv_input(maps_fv, img_feats):
    """the bird's-eye input [B, 2560, 128] of bv_out_layers: [center_fv | cam_offset | img_feats] with H folded into C
    (bev/model.py:190)"""
    return torch.cat([maps_fv, img_feats], 1).reshape(maps_fv.shape[0], -1, 128)


def bv_out(sd, summon):
    """bv_out_layers: 3 x BasicBlock_1D (bev/model.py:191) -> [B, 128, 128] = center_bv | cam_offset_bv"""
    y = summon
    for i in range(3):
        y = block_1d(sd, f"bv_out_layers.{i}.", y)
    return y


def coarse2fine(sd, feat):
    """coarse2fine_localization + fv_conditioned_bv_estimation, bev/model.py:188-215."""
    maps_fv, x = fv_maps(sd, feat)
    center_fv, cam_off = maps_fv[:, :1], maps_fv[:, 1:4]
    y = bv_out(sd, bv_input(maps_fv, x))
    center_bv, cam_off_bv = y[:, :64], y[:, 64:]
    center_3d = center_fv.repeat(1, 64, 1, 1) * center_bv.unsqueeze(2).repeat(1, 1, 128, 1)  # :195-196
    center_3d = block_3d(sd, "center_map_refiner.0.", center_3d.unsqueeze(1)).squeeze(1)     # :206
    cam_3d = sd["coordmap_3d"] + cam_off.unsqueeze(-1).transpose(4, 1).contiguous()           # :209-210
    cam_3d[:, :, :, :, 2] = cam_3d[:, :, :, :, 2] + cam_off_bv.unsqueeze(2).contiguous()      # :212
    cam_3d = block_3d(sd, "cam_map_refiner.0.", cam_3d.unsqueeze(1).transpose(5, 1).squeeze(-1))  # :213
    return center_3d, cam_3d, center_fv


def parse_3d(center_maps_3d, thresh, max_person=64):
    """CenterMap3D.parse_3dcentermap, bev/post_parser.py:44-66.  MaxPool3d(5,1,2) sees [B,64,128,128] as an
    unbatched (C=B,D,H,W) volume; per-depth top-64 then global top-64 == global top-64 (ties: index asc)."""
    cm = _t(center_maps_3d).float()
    m = F.max_pool3d(cm, 5, 1, 2)
    nm = cm * (m == cm).float()
    b, d, h, w = nm.shape
    flat = nm.reshape(b, -1).numpy()
    bi, zyx, sc = [], [], []
    for i in range(b):
        cand = np.nonzero(flat[i] > np.float32(thresh))[0]
        order = cand[np.lexsort((cand, -flat[i, cand].astype(np.float64)))][:max_person]
        for k in order:
            bi.append(i); zyx.append((k // (h * w), (k % (h * w)) // w, k % w)); sc.append(flat[i, k])
    return (torch.tensor(bi, dtype=torch.int64), torch.tensor(zyx, dtype=torch.int64).reshape(-1, 3),
            torch.tensor(np.array(sc, dtype=np.float32)))


def cam_to_centermap_coords(cams, anchor):
    """convert_cam_params_to_centermap_coords + denormalize_center, bev/model.py:89-102."""
    cc = torch.ones_like(cams)
    cc[:, 1:] = cams[:, 1:]
    if len(cams):
        cc[:, 0] = torch.argmin(torch.abs(cams[:, [0]] - anchor[None]), dim=1).float() / 128 * 2.0 - 1.0
    return torch.clamp((cc + 1) / 2 * 128, 1, 127).long()


@torch.no_grad()
def bev_model(sd, frames_nhwc, thresh, center3d_override=None):
    """BEVv1.forward, bev/model.py:232-250.  Returns None when nobody is detected."""
    sd = R.to_torch_sd(sd)
    feat = R.hrnet32_forward(sd, _t(frames_nhwc).float())
    center_3d, cam_3d, center_fv = coarse2fine(sd, feat)
    if center3d_override is not None:
        center_3d = _t(center3d_override).float()
    bi, czyx, conf = parse_3d(center_3d, thresh)
    if len(bi) == 0:
        return None
    cams = cam_3d[bi, :, czyx[:, 0], czyx[:, 1], czyx[:, 2]]                                # :242
    fv = head_block(sd, "param_head.0.0.", feat)                                            # :244
    from romp_b200.synth import bev_cam3dmap_anchor
    cam_czyx = cam_to_centermap_coords(cams.clone(), torch.from_numpy(bev_cam3dmap_anchor()))   # :226
    f = fv[bi, :, cam_czyx[:, 1], cam_czyx[:, 2]] + sd["position_embeddings.weight"][cam_czyx[:, 0]]   # :217-223
    h = F.relu(F.linear(f, sd["transformer.0.weight"], sd["transformer.0.bias"]))
    h = F.relu(F.linear(h, sd["transformer.3.weight"], sd["transformer.3.bias"]))
    p = F.linear(h, sd["transformer.6.weight"], sd["transformer.6.bias"])
    return {"params_pred": torch.cat([cams, p], 1), "cam_czyx": cam_czyx, "pred_batch_ids": bi, "pred_czyxs": czyx,
            "center_confs": conf, "center_map_3d": center_3d, "cam_maps_3d": cam_3d, "center_map": center_fv,
            "front_view_features": fv}


def cam_to_trans(cams):
    """denormalize_cam_params_to_trans, bev/post_parser.py:114-128."""
    cams = _t(cams)
    depth = (1 / (cams[:, 0] * TAN_FOV + 1e-3)).unsqueeze(1)
    xy = torch.flip(cams[:, 1:], [1]) * depth * TAN_FOV
    return torch.cat([xy, depth], 1)


def perspective_project(points, trans, focal=443.4, img=512):
    """perspective_projection, bev/post_parser.py:68-107 (no rotation, no camera centre, normalised)."""
    p = _t(points) + _t(trans).unsqueeze(1)
    p = p / (p[:, :, -1].unsqueeze(-1) + 1e-6)
    K = torch.zeros(p.shape[0], 3, 3)
    K[:, 0, 0] = focal; K[:, 1, 1] = focal; K[:, 2, 2] = 1.0
    return torch.matmul(p.contiguous(), K)[:, :, :-1].contiguous() / (float(img) / 2.0)


def smpla_forward(pack_a, pack_smil, betas, thetas, root_align=True):
    """SMPLA_parser.forward, bev/post_parser.py:255-278: adults SMPL-A (11 betas), babies (betas[:,10] > 0.8) SMIL (10)."""
    betas, thetas = _t(betas).float(), _t(thetas).float()
    n = len(thetas)
    baby = betas[:, 10] > 0.8
    verts, joints = torch.zeros(n, 6890, 3), torch.zeros(n, 71, 3)
    if baby.any():
        v, j = R.smpl_forward(pack_smil, betas[baby, :10], thetas[baby])
        verts[baby], joints[baby] = v, j
    if (~baby).any():
        v, j = R.smpl_forward(pack_a, betas[~baby], thetas[~baby], shape_key="smpla_shapedirs")
        verts[~baby], joints[~baby] = v, j
    if root_align:
        root = joints[:, [45, 46]].mean(1, keepdim=True)
        joints, verts = joints - root, verts - root
    return verts, joints


def suppress_redundant(pj2d, cam, img_shape, thresh):
    """suppressing_redundant_prediction_via_projection, bev/post_parser.py:167-198 -> indices that survive."""
    n = len(pj2d)
    if n == 1:
        return list(range(n))
    pj2d, cam = _t(pj2d), _t(cam)
    dist = torch.norm(pj2d.unsqueeze(1) - pj2d.unsqueeze(0), p=2, dim=-1).mean(-1)
    sc = cam[:, 0] * 2
    mx = torch.max(sc.unsqueeze(1).expand(n, n), sc.unsqueeze(0).expand(n, n))
    dn = dist / mx
    dn[torch.triu(torch.ones_like(dn), diagonal=1) < 0.5] = 10000.0
    thr = thresh * max(img_shape) / 640
    i0, i1 = torch.where(dn < thr)
    removed = torch.where(sc[i0] < sc[i1], i0, i1).tolist()
    return [i for i in range(n) if i not in set(removed)]


def remove_outlier(cam_trans, cam, relative_scale_thresh=3, scale_thresh=0.25):
    """remove_outlier, bev/post_parser.py:200-222 -> indices that survive."""
    cam_trans, cam = _t(cam_trans), _t(cam)
    n = len(cam_trans)
    if n < 3:
        return list(range(n))
    d = torch.norm(cam_trans.unsqueeze(1) - cam_trans.unsqueeze(0), p=2, dim=-1)
    d = torch.sort(d).values[:, 1:-1]
    mean_dist = d.mean(1)
    rel = mean_dist / ((mean_dist.sum() - mean_dist) / (n - 1))
    out = (rel > relative_scale_thresh) & (cam[:, 0] < scale_thresh)
    return [i for i in range(n) if not bool(out[i])]


@torch.no_grad()
def bev_forward(sd, pack_a, pack_smil, frames_nhwc, thresh=0.08, nms_thresh=20, rel_scale_thresh=1.6,
                img_shape=(512, 512), offsets=(0, 512, 0, 512, 512, 512), center3d_override=None):
    """BEV.process_normal_image (bev/main.py:158-181) for ONE frame batch element semantics applied per frame."""
    out = bev_model(sd, frames_nhwc, thresh, center3d_override)
    if out is None:
        return None
    pk = R.pack_params(out["params_pred"], num_betas=11)
    res = {"params_pred": out["params_pred"], "center_confs": out["center_confs"], "pred_batch_ids": out["pred_batch_ids"],
           "cam": pk["cam"], "smpl_thetas": pk["smpl_thetas"], "smpl_betas": pk["smpl_betas"], "cam_trans": cam_to_trans(pk["cam"])}
    verts, joints = smpla_forward(pack_a, pack_smil, res["smpl_betas"], res["smpl_thetas"])
    pj2d = perspective_project(joints, res["cam_trans"])
    # NB the reference maps pj2d to original-image pixels in place (bev/post_parser.py:129-136,150), so its later
    # post-filters see pj2d == pj2d_org
    res.update(verts=verts, joints=joints, pj2d_org=R.to_org_image(pj2d, offsets))
    res["pj2d"] = res["pj2d_org"]
    keep = []
    for b in sorted(set(res["pred_batch_ids"].tolist())):       # the reference post-filters assume one frame
        idx = [i for i, v in enumerate(res["pred_batch_ids"].tolist()) if v == b]
        k1 = [idx[i] for i in suppress_redundant(res["pj2d"][idx], res["cam"][idx], img_shape, nms_thresh)]
        k2 = [k1[i] for i in remove_outlier(res["cam_trans"][k1], res["cam"][k1], rel_scale_thresh)]
        keep += k2
    res = {k: v[keep] for k, v in res.items()}
    res["_model"] = out
    return res
