"""CPU restatement of BEV's long-image (crowd) mode for the tests.  TEST INFRASTRUCTURE ONLY.

bev/split2process.py (padding_image_overlap, get_image_split_plan, exclude_boudary_subjects,
convert_crop_cam_params2full_image, collect_outputs) and the filter stages of BEV.process_long_image (bev/main.py:208-256),
stage by stage, on per-crop outputs (cam, center_confs, betas, thetas, params_pred, verts, joints).  Built on
oracle/bev_oracle.py and pinned by tests/golden/bev_long_post.npz (tests/golden/make_golden_bev_long.py), which runs the
reference's own loop.
"""
from __future__ import annotations

import numpy as np
import torch

from oracle import bev_oracle as B
from oracle import romp_oracle as R


def long_image_plan(h, w, overlap_ratio):
    """-> (pad_length, boxes int32 [K,4] = [left, right, top, bottom], pad_info6).  The last box starts at W - h and keeps
    the previous box's right edge; all boxes are truncated to int32 from float64."""
    pad = int(h * overlap_ratio)
    W = w + 2 * pad
    k = int(np.ceil((W / h - 1) / (1 - overlap_ratio))) + 1
    lefts = [(1 - overlap_ratio) * h * i for i in range(k - 1)]
    rights = [x + h for x in lefts]
    rows = [[x, r, 0, h] for x, r in zip(lefts, rights)] + [[W - h, rights[-1], 0, h]]
    top = (w - h) // 2
    return pad, np.asarray(rows, dtype=np.float64).astype(np.int32), np.array([top, w - top, 0, w, h, w], np.float32)


def suppress_conf(pj2d, cam, conf, img_shape, thresh):
    """suppressing_redundant_prediction_via_projection(conf_based=True), bev/post_parser.py:167-198 -> surviving indices.
    Every pair below the threshold at once; of a pair the lower center_confs goes, on a tie the later one."""
    n = len(pj2d)
    if n == 1:
        return [0]
    pj2d, cam, conf = R._t(pj2d), R._t(cam), R._t(conf)
    dist = torch.norm(pj2d.unsqueeze(1) - pj2d.unsqueeze(0), p=2, dim=-1).mean(-1)
    sc = cam[:, 0] * 2
    dn = dist / torch.max(sc.unsqueeze(1).expand(n, n), sc.unsqueeze(0).expand(n, n))
    dn[torch.triu(torch.ones_like(dn), diagonal=1) < 0.5] = 10000.0
    i0, i1 = torch.where(dn < thresh * max(img_shape) / 640)
    removed = set(torch.where(conf[i0] < conf[i1], i0, i1).tolist())
    return [i for i in range(n) if i not in removed]


def project(joints, cam, offsets):
    trans = B.cam_to_trans(cam)
    return trans, R.to_org_image(B.perspective_project(joints, trans), offsets)


def long_image_post(crops, boxes, pad_length, h, w, nms_thresh=20.0, rel_scale_thresh=1.6):
    """Steps 3-7 of the long-image mode.  crops[i]: None (nothing detected) or a dict of torch tensors with cam [n,3],
    center_confs [n], smpl_betas [n,11], smpl_thetas [n,72], params_pred [n,146], verts [n,6890,3], joints [n,71,3].

    Returns (stages, out): stages[i] = dict of crop-local survivor indices after the boundary drop ("boundary"), the
    suppression ("nms") and remove_outlier ("outlier"); stages["merged_nms"] / ["final"] index the concatenated
    survivors; out = the final dict (pred_batch_ids all zero).  Each crop uses its own box geometry."""
    k = len(boxes)
    ratio = [(int(boxes[i, 1]) - int(boxes[i + 1, 0])) / h / 2 for i in range(k - 1)]
    stages, rows = {}, []
    for i, c in enumerate(crops):
        if c is None:
            continue
        l, r, t, b = (int(v) for v in boxes[i])
        ch, cw = b - t, r - l
        x = c["cam"][:, 2]
        drop = torch.zeros(len(x), dtype=torch.bool)
        if i != k - 1:
            drop |= x > (1 - ratio[i])
        if i >= 2:
            drop |= x < (ratio[i - 1] - 1)
        idx = torch.where(~drop)[0].tolist()
        cam = c["cam"][idx]
        trans, pj = project(c["joints"][idx], cam, [0, ch, 0, cw, ch, cw])
        k1 = suppress_conf(pj, cam, c["center_confs"][idx], [ch, cw], nms_thresh) if idx else []
        k2 = [k1[j] for j in B.remove_outlier(trans[k1], cam[k1], rel_scale_thresh, scale_thresh=1)]
        stages[i] = {"boundary": idx, "nms": [idx[j] for j in k1], "outlier": [idx[j] for j in k2]}
        keep = stages[i]["outlier"]
        cam_full = c["cam"][keep].clone()
        cam_full *= np.float64(max(r - l, b - t) / max(h, w))                        # split2process.py:51-52
        cam_full[:, 2] += np.float64(((l - pad_length) + (r - pad_length)) / 2 / (w / 2) - 1)   # :56-57
        rows.append({"cam": cam_full, "center_confs": c["center_confs"][keep], "smpl_betas": c["smpl_betas"][keep],
                     "smpl_thetas": c["smpl_thetas"][keep], "params_pred": c["params_pred"][keep], "verts": c["verts"][keep],
                     "joints": c["joints"][keep], "crop": torch.full((len(keep),), i, dtype=torch.int64),
                     "index": torch.tensor(keep, dtype=torch.int64)})
    if not rows:
        return stages, None
    m = {key: torch.cat([r_[key] for r_ in rows], 0) for key in rows[0]}
    top = (w - h) // 2
    trans, pj = project(m["joints"], m["cam"], [top, w - top, 0, w, h, w])
    k1 = suppress_conf(pj, m["cam"], m["center_confs"], (h, w, 3), nms_thresh) if len(pj) else []
    k2 = [k1[j] for j in B.remove_outlier(trans[k1], m["cam"][k1], rel_scale_thresh, scale_thresh=0.5)]
    stages["merged_nms"], stages["final"] = k1, k2
    out = {"smpl_thetas": m["smpl_thetas"][k2], "smpl_betas": m["smpl_betas"][k2], "cam": m["cam"][k2], "cam_trans": trans[k2],
           "params_pred": m["params_pred"][k2], "center_confs": m["center_confs"][k2],
           "pred_batch_ids": torch.zeros(len(k2), dtype=torch.int64), "verts": m["verts"][k2], "joints": m["joints"][k2],
           "pj2d_org": pj[k2], "crop": m["crop"][k2], "index": m["index"][k2]}
    return stages, out


def planted_volumes(n, seed):
    """Per-crop 3-D centre maps for the end-to-end long-image tests: uniform noise below 0.05 and 1-4 planted centres per
    crop, spaced >= 3 voxels apart, with confidences in [0.2, 1) that are distinct across the whole image."""
    rs = np.random.RandomState(seed)
    vol = rs.uniform(0, 0.05, size=(n, 64, 128, 128)).astype(np.float32)
    used = set()
    for b in range(n):
        cells = []
        for _ in range(rs.randint(1, 5)):
            z, y, x = rs.randint(0, 64), rs.randint(16, 112), rs.randint(8, 120)
            if all(max(abs(z - c[0]), abs(y - c[1]), abs(x - c[2])) >= 3 for c in cells):
                cells.append((z, y, x))
        for z, y, x in cells:
            v = np.float32(rs.uniform(0.2, 1.0))
            while v in used:
                v = np.float32(rs.uniform(0.2, 1.0))
            used.add(v)
            vol[b, z, y, x] = v
    return vol


def long_image(h, w, seed):
    """Seeded BGR test image."""
    return np.random.RandomState(seed).randint(0, 256, size=(h, w, 3)).astype(np.uint8)
