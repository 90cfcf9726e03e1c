"""CPU oracle for the ROMP per-frame inference hot path.  TEST INFRASTRUCTURE ONLY.

This is a from-scratch fp32 CPU restatement (torch CPU ops / numpy, functional style, driven by a flat
state dict) of the reference algorithm.  Only ``tests/``, ``__graft_entry__.smoke()`` and the
``cpu_baseline`` / ``--impl reference`` legs of ``bench.py`` may import it; the product package
``romp_b200`` never does.

Parity pin: every function below is checked against the *reference's own code* imported from
``/root/reference/simple_romp`` in the build container (``tests/golden/make_golden.py`` writes the
fixtures in ``tests/golden/``; ``tests/test_oracle_golden.py`` replays them anywhere, and
``tests/test_oracle_vs_reference.py`` re-runs the live comparison whenever ``/root/reference`` exists).
The reference ships no golden vectors or unit tests for this path (SURVEY section 4), so the fixtures
generated from the reference code are the pin.  ``cam_trans`` from ``cv2.solvePnPRansac`` is
"parity unpinned" beyond a loose tolerance (RANSAC); the closed-form least squares
(`estimate_translation_lsq`) follows the reference's own fallback and is pinned tightly.

Each function cites the reference file:line it restates.
"""
from __future__ import annotations

import math

import numpy as np
import torch
import torch.nn.functional as F

BN_EPS = 1e-5  # torch.nn.BatchNorm2d default used throughout simple_romp/romp/model.py


def _t(x):
    return x if isinstance(x, torch.Tensor) else torch.from_numpy(np.asarray(x))


def to_torch_sd(sd):
    return {k: _t(v) for k, v in sd.items()}


# ----------------------------------------------------------------------------------------------
# a2-a5: backbone + head  (simple_romp/romp/model.py)
# ----------------------------------------------------------------------------------------------
# Operand rounding of every convolution.  None = the reference's CPU arithmetic (fp32).  "tf32" = what the reference's
# default GPU path computes (SURVEY 8a3: torch.backends.cudnn.allow_tf32 is True and the reference never touches it, so
# cuDNN runs the convs on TF32 tensor cores): both conv operands rounded to 10 mantissa bits, round-to-nearest with ties
# away from zero (cvt.rna.tf32.f32), fp32 accumulation, everything else (BatchNorm, residual adds, upsampling) in fp32.
# This "oracle under TF32-equivalent rounding" gives the error of the reference's own GPU arithmetic against its CPU
# arithmetic - the yardstick for the tensor-core engines.
CONV_OPERAND_ROUNDING = None


def round_tf32(x):
    """fp32 -> TF32 (10-bit mantissa), ties away from zero; values stay in fp32 containers."""
    i = x.contiguous().view(torch.int32)
    return ((i + 0x1000) & ~0x1FFF).view(torch.float32)


class conv_rounding:
    """with conv_rounding("tf32"): ...  - run oracle convolutions with TF32-rounded operands."""

    def __init__(self, mode):
        assert mode in (None, "tf32")
        self.mode = mode

    def __enter__(self):
        global CONV_OPERAND_ROUNDING
        self.prev, CONV_OPERAND_ROUNDING = CONV_OPERAND_ROUNDING, self.mode

    def __exit__(self, *exc):
        global CONV_OPERAND_ROUNDING
        CONV_OPERAND_ROUNDING = self.prev


def _conv2d(x, w, b, stride, padding):
    if CONV_OPERAND_ROUNDING == "tf32":
        x, w = round_tf32(x), round_tf32(w)
    return F.conv2d(x, w, b, stride=stride, padding=padding)


def conv_bn(sd, conv, bn, x, stride=1, relu=False):
    """Conv2d(k, stride, pad=k//2) [+bias] -> eval BatchNorm2d -> optional ReLU (model.py:49-52,70-72)."""
    w = sd[conv + ".weight"]
    b = sd.get(conv + ".bias")
    y = _conv2d(x, w, b, stride, w.shape[-1] // 2)
    if bn is not None:
        y = F.batch_norm(y, sd[bn + ".running_mean"], sd[bn + ".running_var"],
                         sd[bn + ".weight"], sd[bn + ".bias"], False, 0.0, BN_EPS)
    return F.relu(y) if relu else y


def basic_block(sd, p, x):
    """model.py:54-83 (no downsample is ever configured for BasicBlocks in HRNet-32 / ROMP heads)."""
    y = conv_bn(sd, p + "conv1", p + "bn1", x, relu=True)
    y = conv_bn(sd, p + "conv2", p + "bn2", y)
    return F.relu(y + x)


def bottleneck(sd, p, x):
    """model.py:85-123."""
    y = conv_bn(sd, p + "conv1", p + "bn1", x, relu=True)
    y = conv_bn(sd, p + "conv2", p + "bn2", y, relu=True)
    y = conv_bn(sd, p + "conv3", p + "bn3", y)
    res = x
    if (p + "downsample.0.weight") in sd:
        res = conv_bn(sd, p + "downsample.0", p + "downsample.1", x)
    return F.relu(y + res)


def hr_module(sd, p, xs, channels, multi_scale_output=True):
    """HighResolutionModule.forward, model.py:226-244, fuse layers :178-221."""
    nb = len(channels)
    xs = list(xs)
    for b in range(nb):
        for k in range(4):
            xs[b] = basic_block(sd, f"{p}branches.{b}.{k}.", xs[b])
    outs = []
    for i in range(nb if multi_scale_output else 1):
        y = None
        for j in range(nb):
            q = f"{p}fuse_layers.{i}.{j}."
            if j == i:
                t = xs[j]
            elif j > i:
                t = conv_bn(sd, q + "0", q + "1", xs[j])
                t = F.interpolate(t, scale_factor=2 ** (j - i), mode="nearest")
            else:
                t = xs[j]
                for k in range(i - j):
                    t = conv_bn(sd, f"{q}{k}.0", f"{q}{k}.1", t, stride=2, relu=(k != i - j - 1))
            y = t if y is None else y + t
        outs.append(F.relu(y))
    return outs


def hrnet32_forward(sd, frames_nhwc):
    """HigherResolutionNet.forward, model.py:382-417.  frames: [B,512,512,3] float 0..255 (RGB)."""
    x = frames_nhwc.permute(0, 3, 1, 2)
    x = ((x / 255.0) * 2.0 - 1.0).contiguous()
    p = "backbone."
    x = conv_bn(sd, p + "conv1", p + "bn1", x, stride=2, relu=True)
    x = conv_bn(sd, p + "conv2", p + "bn2", x, stride=2, relu=True)
    for i in range(4):
        x = bottleneck(sd, f"{p}layer1.{i}.", x)
    xs = [conv_bn(sd, p + "transition1.0.0", p + "transition1.0.1", x, relu=True),
          conv_bn(sd, p + "transition1.1.0.0", p + "transition1.1.0.1", x, stride=2, relu=True)]
    ys = hr_module(sd, p + "stage2.0.", xs, [32, 64])
    xs = [ys[0], ys[1],
          conv_bn(sd, p + "transition2.2.0.0", p + "transition2.2.0.1", ys[-1], stride=2, relu=True)]
    for m in range(4):
        xs = hr_module(sd, f"{p}stage3.{m}.", xs, [32, 64, 128])
    ys = xs
    xs = [ys[0], ys[1], ys[2],
          conv_bn(sd, p + "transition3.3.0.0", p + "transition3.3.0.1", ys[-1], stride=2, relu=True)]
    for m in range(3):
        xs = hr_module(sd, f"{p}stage4.{m}.", xs, [32, 64, 128, 256], multi_scale_output=(m != 2))
    return xs[0]


def coord_maps(size=128, dtype=torch.float32):
    """get_coord_maps, model.py:8-37: ch0 varies along W, ch1 along H, value i/(size-1)*2-1 (computed in `dtype`)."""
    r = torch.arange(size, dtype=dtype) / (size - 1) * 2 - 1
    xx = r.view(1, 1, 1, size).expand(1, 1, size, size)
    yy = r.view(1, 1, size, 1).expand(1, 1, size, size)
    return torch.cat([xx, yy], 1).contiguous()


def romp_head(sd, feat):
    """ROMPv1.forward after the backbone, model.py:470-481 (+ head layout :445-468)."""
    cm = coord_maps(128, torch.promote_types(feat.dtype, torch.float32))     # fp32, or float64 for float64 features
    x = torch.cat([feat, cm.to(feat.device).expand(feat.shape[0], -1, -1, -1)], 1)
    outs = {}
    for h in (1, 2, 3):
        q = f"final_layers.{h}."
        y = conv_bn(sd, q + "0.0", q + "0.1", x, stride=2, relu=True)
        for blk in range(2):
            y = basic_block(sd, f"{q}1.{blk}.0.", y)
        outs[h] = conv_bn(sd, q + "2", None, y)
    center_maps = outs[2]
    params_maps = torch.cat([outs[3], outs[1]], 1)
    return center_maps, params_maps


@torch.no_grad()
def romp_maps(sd, frames_nhwc, dtype=torch.float32):
    """Seam S1 (`self.model(x)`, main.py:112) followed by the cam-scale pow of main.py:113, in `dtype` (that of sd)."""
    sd = to_torch_sd(sd)
    center, params = romp_head(sd, hrnet32_forward(sd, _t(frames_nhwc).to(dtype)))
    params = params.clone()
    params[:, 0] = torch.pow(1.1, params[:, 0])
    return center, params


# ----------------------------------------------------------------------------------------------
# a7-a9: center-map parse  (simple_romp/romp/post_parser.py:27-64,128-146; SURVEY appendix C)
# ----------------------------------------------------------------------------------------------
def nms5(center_maps):
    """post_parser.py:50-54 with MaxPool2d(5,1,2) (:24): det * float(maxpool(det) == det)."""
    m = F.max_pool2d(center_maps, 5, 1, 2)
    return center_maps * (m == center_maps).float()


def parse_centermap(center_maps, thresh=0.25, max_person=64):
    """post_parser.py:27-47.  Deterministic tie rule: score desc, then flat index asc.

    Returns batch_ids[N] i64, flat_inds[N] i64, center_yxs[N,2] f32, scores[N] f32; persons ordered by
    (batch asc, score desc) exactly like ``torch.where(mask)`` on the [B,K] score table.
    """
    cm = nms5(_t(center_maps).float())
    b, c, h, w = cm.shape
    assert c == 1
    flat = cm.reshape(b, -1).numpy()
    bi, fi, sc = [], [], []
    for i in range(b):
        order = np.lexsort((np.arange(flat.shape[1]), -flat[i].astype(np.float64)))[:max_person]
        for k in order:
            if flat[i, k] > np.float32(thresh):
                bi.append(i); fi.append(int(k)); sc.append(flat[i, k])
    batch_ids = torch.tensor(bi, dtype=torch.int64)
    flat_inds = torch.tensor(fi, dtype=torch.int64)
    scores = torch.tensor(np.array(sc, dtype=np.float32))
    yxs = torch.stack([(flat_inds // w).float(), (flat_inds % w).float()], 1) if len(bi) else torch.zeros(0, 2)
    return batch_ids, flat_inds, yxs, scores


def parameter_sampling(maps, batch_ids, flat_inds):
    """post_parser.py:128-133: maps[B,C,H,W] -> [N,C] rows at (batch, flat pixel)."""
    maps = _t(maps)
    b, c = maps.shape[:2]
    return maps.reshape(b, c, -1)[batch_ids, :, flat_inds].contiguous()


# ----------------------------------------------------------------------------------------------
# a10-a11: parameter unpack and 6D -> axis-angle  (post_parser.py:66-79, utils.py:471-682)
# ----------------------------------------------------------------------------------------------
def rot6d_to_rotmat(x):
    """utils.py:477-491."""
    x = x.reshape(-1, 3, 2)
    b1 = F.normalize(x[:, :, 0], dim=1, eps=1e-6)
    dot = torch.sum(b1 * x[:, :, 1], dim=1, keepdim=True)
    b2 = F.normalize(x[:, :, 1] - dot * b1, dim=-1, eps=1e-6)
    b3 = torch.cross(b1, b2, dim=1)
    return torch.stack([b1, b2, b3], dim=-1)


def rotmat_to_quat(R, eps=1e-6):
    """utils.py:606-682 (kornia lineage): 4-branch select on the transposed matrix."""
    Rt = R.transpose(1, 2)
    m = lambda i, j: Rt[:, i, j]
    d2 = m(2, 2) < eps
    d01 = m(0, 0) > m(1, 1)
    d0n1 = m(0, 0) < -m(1, 1)
    t0 = 1 + m(0, 0) - m(1, 1) - m(2, 2)
    q0 = torch.stack([m(1, 2) - m(2, 1), t0, m(0, 1) + m(1, 0), m(2, 0) + m(0, 2)], -1)
    t1 = 1 - m(0, 0) + m(1, 1) - m(2, 2)
    q1 = torch.stack([m(2, 0) - m(0, 2), m(0, 1) + m(1, 0), t1, m(1, 2) + m(2, 1)], -1)
    t2 = 1 - m(0, 0) - m(1, 1) + m(2, 2)
    q2 = torch.stack([m(0, 1) - m(1, 0), m(2, 0) + m(0, 2), m(1, 2) + m(2, 1), t2], -1)
    t3 = 1 + m(0, 0) + m(1, 1) + m(2, 2)
    q3 = torch.stack([t3, m(1, 2) - m(2, 1), m(2, 0) - m(0, 2), m(0, 1) - m(1, 0)], -1)
    c0 = (d2 & d01).float().unsqueeze(1)
    c1 = (d2 & ~d01).float().unsqueeze(1)
    c2 = (~d2 & d0n1).float().unsqueeze(1)
    c3 = (~d2 & ~d0n1).float().unsqueeze(1)
    q = q0 * c0 + q1 * c1 + q2 * c2 + q3 * c3
    q = q / torch.sqrt(t0.unsqueeze(1) * c0 + t1.unsqueeze(1) * c1 + t2.unsqueeze(1) * c2 + t3.unsqueeze(1) * c3)
    return q * 0.5


def quat_to_aa(q):
    """utils.py:554-604 and the NaN->0 of :551."""
    q1, q2, q3 = q[:, 1], q[:, 2], q[:, 3]
    s2 = q1 * q1 + q2 * q2 + q3 * q3
    s = torch.sqrt(s2)
    c = q[:, 0]
    two_theta = 2.0 * torch.where(c < 0.0, torch.atan2(-s, -c), torch.atan2(s, c))
    k = torch.where(s2 > 0.0, two_theta / s, 2.0 * torch.ones_like(s))
    aa = torch.stack([q1 * k, q2 * k, q3 * k], 1)
    aa[torch.isnan(aa)] = 0.0
    return aa


def rotmat_to_aa(Rm):
    """rotation_matrix_to_angle_axis, utils.py:535-552: [N,3,3] -> [N,3]."""
    return quat_to_aa(rotmat_to_quat(Rm))


def rot6d_to_aa(x6):
    """rot6D_to_angular, utils.py:471-475: [N, J*6] -> [N, J*3]."""
    n = x6.shape[0]
    return quat_to_aa(rotmat_to_quat(rot6d_to_rotmat(x6))).reshape(n, -1)


def pack_params(params_pred, num_betas=10):
    """pack_params_dict, post_parser.py:66-79 (BEV: bev/post_parser.py:240-253 with 11 betas)."""
    p = _t(params_pred).float()
    n = p.shape[0]
    cam, go6, bp6, betas = p[:, :3], p[:, 3:9], p[:, 9:135], p[:, 135:135 + num_betas]
    body = torch.cat([rot6d_to_aa(bp6.contiguous()), torch.zeros(n, 6)], 1)
    go = rot6d_to_aa(go6.contiguous())
    return {"cam": cam.contiguous(), "global_orient": go, "body_pose": body,
            "smpl_betas": betas.contiguous(), "smpl_thetas": torch.cat([go, body], 1)}


def parsing_outputs(center_maps, params_maps, thresh=0.25):
    """post_parser.py:135-146; returns None when nobody is detected."""
    batch_ids, flat_inds, yxs, scores = parse_centermap(center_maps, thresh)
    if len(batch_ids) == 0:
        return None
    params_pred = parameter_sampling(params_maps, batch_ids, flat_inds)
    out = pack_params(params_pred)
    out["params_pred"] = params_pred
    out["pred_batch_ids"] = batch_ids
    out["flat_inds"] = flat_inds
    out["center_preds"] = torch.stack([flat_inds % 64, flat_inds // 64], 1) * 512 // 64
    out["center_confs"] = parameter_sampling(center_maps, batch_ids, flat_inds)
    return out


# ----------------------------------------------------------------------------------------------
# a13-a16: SMPL forward  (simple_romp/romp/smpl.py:24-35,62-290; SURVEY appendix D)
# ----------------------------------------------------------------------------------------------
def batch_rodrigues(rv, dtype=torch.float32, device="cpu"):
    """smpl.py:191-222.  NB eps is added to every component before the norm (:206).  ``dtype`` / ``device``: where and in
    which precision to compute (the defaults are the reference's CPU fp32 arithmetic)."""
    rv = _t(rv).to(device=device, dtype=dtype)
    angle = torch.norm(rv + 1e-8, dim=1, keepdim=True)
    d = rv / angle
    c, s = torch.cos(angle)[:, :, None], torch.sin(angle)[:, :, None]
    rx, ry, rz = d[:, 0:1], d[:, 1:2], d[:, 2:3]
    z = torch.zeros_like(rx)
    K = torch.cat([z, -rz, ry, rz, z, -rx, -ry, rx, z], 1).view(-1, 3, 3)
    return torch.eye(3, dtype=dtype, device=device).unsqueeze(0) + s * K + (1 - c) * torch.bmm(K, K)


def smpl_forward(pack, betas, thetas, root_align=False, shape_key="shapedirs", dtype=torch.float32, device="cpu",
                 stages=False):
    """SMPL.forward + lbs + batch_rigid_transform + VertexJointSelector (smpl.py:62-108,111-188,236-290,24-35).

    Returns verts [N,6890,3], joints71 [N,71,3] (24 SMPL + 21 picked verts + 9 + 17 regressed).  ``dtype`` / ``device``:
    the precision and device of every operation (the defaults are the reference's CPU fp32 arithmetic).  With ``stages``
    a third result holds the intermediate stages: "feat" [N, n_betas+207] = [betas | (R[1:]-I)], "A" [N,24,3,4] (the
    relative transforms), "v_posed" [N,6890,3], "T" [N,6890,4,4] (the blended transforms) and "J_regressed" [N,24,3]
    (the rest-pose joints).
    """
    pk = {k: _t(v) for k, v in pack.items()}
    fl = lambda x: x.to(device=device, dtype=dtype)
    betas, thetas = fl(_t(betas)), fl(_t(thetas))
    n = betas.shape[0]
    vt, sdirs, pdirs = fl(pk["v_template"]), fl(pk[shape_key]), fl(pk["posedirs"])
    Jr, W, parents = fl(pk["J_regressor"]), fl(pk["weights"]), pk["kintree_table"].tolist()
    eye3 = torch.eye(3, dtype=dtype, device=device)
    v_shaped = vt.unsqueeze(0) + torch.einsum("bl,mkl->bmk", betas, sdirs)                 # :153
    J = torch.einsum("bik,ji->bjk", v_shaped, Jr)                                           # :156
    R = batch_rodrigues(thetas.reshape(-1, 3), dtype, device).view(n, 24, 3, 3)            # :163
    pf = (R[:, 1:] - eye3).reshape(n, 207)                                                  # :165
    v_posed = v_shaped + torch.matmul(pf, pdirs).view(n, -1, 3)                             # :167-170
    rel = J.clone()
    rel[:, 1:] = J[:, 1:] - J[:, parents[1:]]                                               # :262-263
    L = torch.zeros(n, 24, 4, 4, dtype=dtype, device=device)
    L[:, :, :3, :3] = R
    L[:, :, :3, 3] = rel
    L[:, :, 3, 3] = 1.0                                                                     # :224-234
    G = [L[:, 0]]
    for i in range(1, 24):
        G.append(torch.matmul(G[parents[i]], L[:, i]))                                      # :270-275
    G = torch.stack(G, 1)
    J_posed = G[:, :, :3, 3]                                                                # :280
    Jh = torch.cat([J, torch.zeros(n, 24, 1, dtype=dtype, device=device)], 2).unsqueeze(-1)
    A = G.clone()
    A[:, :, :, 3] = G[:, :, :, 3] - torch.matmul(G, Jh)[..., 0]                             # :285-288
    T = torch.matmul(W.unsqueeze(0).expand(n, -1, -1), A.view(n, 24, 16)).view(n, -1, 4, 4)  # :176-180
    vh = torch.cat([v_posed, torch.ones(n, v_posed.shape[1], 1, dtype=dtype, device=device)], 2).unsqueeze(-1)
    verts = torch.matmul(T, vh)[:, :, :3, 0]                                                # :182-186
    j21 = verts[:, pk["extra_joints_index"].to(device)]
    j9 = torch.einsum("bik,ji->bjk", verts, fl(pk["J_regressor_extra9"]))
    j17 = torch.einsum("bik,ji->bjk", verts, fl(pk["J_regressor_h36m17"]))
    joints = torch.cat([J_posed, j21, j9, j17], 1)                                          # :25-29
    if root_align:                                                                          # :102-106
        root = joints[:, [45, 46]].mean(1, keepdim=True)
        joints, verts = joints - root, verts - root
    if stages:
        feat = torch.cat([betas, pf], 1)
        return verts, joints, {"feat": feat, "A": A[:, :, :3, :], "v_posed": v_posed, "T": T, "J_regressed": J}
    return verts, joints


# ----------------------------------------------------------------------------------------------
# a12, a17, a18: camera conversion and projection (utils.py:303-315,347-389; post_parser.py:81-114)
# ----------------------------------------------------------------------------------------------
def cam_to_trans(cam, weight=2.0):
    """convert_cam_to_3d_trans, utils.py:303-307."""
    cam = _t(cam)
    s, tx, ty = cam[:, 0], cam[:, 1], cam[:, 2]
    return torch.stack([tx / s, ty / s, 1.0 / s], 1) * weight


def orth_project(X, cam, keep_dim=False):
    """batch_orth_proj, utils.py:309-315."""
    X, cam = _t(X), _t(cam).view(-1, 1, 3)
    out = X[:, :, :2] * cam[:, :, 0:1] + cam[:, :, 1:]
    if keep_dim:
        out = torch.cat([out, X[:, :, 2:3]], -1)
    return out


def to_org_image(kps, offsets):
    """convert_proejection_from_input_to_orgimg, post_parser.py:81-88.  Returns a NEW tensor; the reference mutates its
    argument in place, so that in its output dict `pj2d` aliases `pj2d_org` - BEV's duplicate-suppression filter
    (bev/post_parser.py:167-198) is called with that aliased tensor, i.e. with original-image pixels; csrc/bev.cu and
    oracle/bev_oracle.py honour this by feeding the filter `pj2d_org`."""
    top, bottom, left, right, h, w = [float(v) for v in offsets]
    size = max(h, w)
    out = _t(kps).clone()
    out[:, :, 0] = (out[:, :, 0] + 1) * size / 2 - left
    out[:, :, 1] = (out[:, :, 1] + 1) * size / 2 - top
    if out.shape[-1] == 3:
        out[:, :, 2] = (out[:, :, 2] + 1) * size / 2
    return out


def estimate_translation_lsq(j3d, j2d, focal=443.4, img=512.0):
    """estimate_translation (utils.py:391-436) with the closed-form solver estimate_translation_np
    (:347-389, unit weights) in place of cv2.solvePnPRansac: validity mask of :404-408,419 (2-D y > -2 and
    3-D z != -2), fewer than 4 valid joints -> INVALID_TRANS = -1 (:420-422); float64 normal equations."""
    j3d32, j2d32 = np.asarray(j3d, np.float32), np.asarray(j2d, np.float32)
    out = np.zeros((j3d32.shape[0], 3), np.float32)
    for i in range(j3d32.shape[0]):
        valid = (j2d32[i, :, -1] > -2.0) & (j3d32[i, :, -1] != -2.0)
        if valid.sum() < 4:
            out[i] = -1.0
            continue
        p3, p2 = j3d32[i][valid].astype(np.float64), j2d32[i][valid].astype(np.float64)
        n = p3.shape[0]
        Z = np.repeat(p3[:, 2], 2)
        XY = p3[:, :2].reshape(-1)
        O = np.tile(np.array([img / 2, img / 2]), n)
        Fv = np.full(2 * n, focal)
        Q = np.stack([Fv * np.tile([1, 0], n), Fv * np.tile([0, 1], n), O - p2.reshape(-1)], 1)
        c = (p2.reshape(-1) - O) * Z - Fv * XY
        out[i] = np.linalg.solve(Q.T @ Q, Q.T @ c)
    return out


def project_outputs(joints, verts, cam, offsets):
    """body_mesh_projection2image, post_parser.py:104-114, with cam_trans by closed-form LSQ."""
    pj2d = orth_project(joints, cam)
    j2d_px = (pj2d[:, :24].numpy() + 1) * 256                                               # :98
    cam_trans = estimate_translation_lsq(_t(joints)[:, :24].numpy(), j2d_px)
    out = {"pj2d": pj2d, "cam_trans": torch.from_numpy(cam_trans),
           "pj2d_org": to_org_image(pj2d, offsets)}
    if verts is not None:
        vc = orth_project(verts, cam, keep_dim=True)
        out["verts_camed"] = vc
        out["verts_camed_org"] = to_org_image(vc, offsets)
    return out


# ----------------------------------------------------------------------------------------------
# whole path (ROMP.forward, main.py:160-176) on a batch of already-preprocessed 512x512 frames
# ----------------------------------------------------------------------------------------------
@torch.no_grad()
def romp_forward(sd, pack, frames_nhwc, thresh=0.25, root_align=False, center_override=None):
    center, params = romp_maps(sd, frames_nhwc)
    if center_override is not None:
        center = _t(center_override).float()
    out = parsing_outputs(center, params, thresh)
    if out is None:
        return None
    verts, joints = smpl_forward(pack, out["smpl_betas"], out["smpl_thetas"], root_align)
    out["verts"], out["joints"] = verts, joints
    offsets = [0, 512, 0, 512, 512, 512]
    out.update(project_outputs(joints, verts, out["cam"], offsets))
    out["center_maps"], out["params_maps"] = center, params
    return out


def mpjpe_mm(j_a, j_b):
    """Pelvis-aligned MPJPE over the 24 SMPL joints in mm (romp/lib/loss_funcs/keypoints_loss.py:64-82)."""
    a, b = _t(j_a)[:, :24].double(), _t(j_b)[:, :24].double()
    a = a - a[:, :1]
    b = b - b[:, :1]
    return float(torch.norm(a - b, dim=-1).mean() * 1000.0)


# ----------------------------------------------------------------------------------------------
# cfg1: ROMP with the ResNet-50 backbone (romp/lib/models/resnet_50.py:19-120) - CPU reference plumbing only
# ----------------------------------------------------------------------------------------------
def resnet50_forward(sd, frames_nhwc):
    """ResNet_50.forward (:55-63): /255 + ImageNet mean/std (:32-38), 7x7 s2 stem, maxpool 3x3 s2, [3,4,6,3] bottlenecks
    (stride on the 3x3 conv), three ConvTranspose2d(4,2,1)+BN+ReLU 2048->256->128->64.  -> [B,64,128,128]."""
    x = frames_nhwc.permute(0, 3, 1, 2) / 255.0
    mean = torch.tensor([0.485, 0.456, 0.406]).view(1, 3, 1, 1)
    std = torch.tensor([0.229, 0.224, 0.225]).view(1, 3, 1, 1)
    x = (x - mean) / std
    p = "backbone."
    w = sd[p + "conv1.weight"]
    x = F.conv2d(x, w, None, 2, 3)
    x = F.relu(F.batch_norm(x, sd[p + "bn1.running_mean"], sd[p + "bn1.running_var"], sd[p + "bn1.weight"], sd[p + "bn1.bias"], False, 0.0, BN_EPS))
    x = F.max_pool2d(x, 3, 2, 1)
    for li, blocks in enumerate((3, 4, 6, 3), start=1):
        for b in range(blocks):
            q = f"{p}layer{li}.{b}."
            stride = 2 if (li > 1 and b == 0) else 1
            y = conv_bn(sd, q + "conv1", q + "bn1", x, relu=True)
            y = conv_bn(sd, q + "conv2", q + "bn2", y, stride=stride, relu=True)
            y = conv_bn(sd, q + "conv3", q + "bn3", y)
            res = x
            if (q + "downsample.0.weight") in sd:
                res = conv_bn(sd, q + "downsample.0", q + "downsample.1", x, stride=stride)
            x = F.relu(y + res)
    for i in range(3):
        x = F.conv_transpose2d(x, sd[f"{p}deconv_layers.{3 * i}.weight"], None, stride=2, padding=1)
        bn = f"{p}deconv_layers.{3 * i + 1}"
        x = F.relu(F.batch_norm(x, sd[bn + ".running_mean"], sd[bn + ".running_var"], sd[bn + ".weight"], sd[bn + ".bias"], False, 0.0, BN_EPS))
    return x


@torch.no_grad()
def romp_resnet50_maps(sd, frames_nhwc, dtype=torch.float32):
    """ROMP head (same layout as ROMPv1, 64+2 input channels) on the ResNet-50 features + cam-scale pow, in `dtype`
    (that of sd)."""
    sd = to_torch_sd(sd)
    center, params = romp_head(sd, resnet50_forward(sd, _t(frames_nhwc).to(dtype)))
    params = params.clone()
    params[:, 0] = torch.pow(1.1, params[:, 0])
    return center, params
