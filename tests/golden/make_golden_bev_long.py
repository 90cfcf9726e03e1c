"""Golden fixtures for BEV's long-image (crowd) mode, produced by running the REFERENCE's own BEV.process_long_image loop
(build container only):    python tests/golden/make_golden_bev_long.py

bev/main.py is NOT imported: importing it evaluates ``bev_settings([])``, which downloads a checkpoint when none is
cached.  Instead its source is parsed with ``ast`` and only the two methods ``BEV.process_long_image`` and
``BEV.single_image_forward`` are compiled, with the reference's own post_parser / split2process / img_preprocess
functions as globals, and called with a stub ``self``.  Nothing from the reference's sources is copied - only its
outputs are stored.

  bev_long_post.npz   stage level: synthetic per-crop outputs of a 256x512 image (14 crops) that make every filter rule
                      fire (left / right boundary trim, per-crop suppression incl. a confidence tie, per-crop outlier,
                      merged suppression across neighbouring crops, merged outlier); the survivors after every stage and
                      the final dict.  Plus the crop plans of several image sizes.
  bev_long_model.npz  end to end: a seeded 256x512 BGR image through the reference BEVv1 (synthetic weights) with a
                      planted 3-D centre map per crop; every filter decision clears its threshold by a margin.
"""
import ast
import functools
import os
import sys
import tempfile
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)
from make_golden import REF, load_reference  # noqa: E402

H, W = 256, 512
PLAN_SIZES = [(256, 512), (256, 600), (480, 2000), (960, 1920), (1080, 3840), (300, 1000)]
MARGIN_X, MARGIN_REL = 0.02, 0.05


class Recorder:
    """Wraps the reference's filters: records the person ids entering / leaving every call and checks the margins."""

    def __init__(self, PP, SP, check_margins):
        self.PP, self.SP, self.calls, self.check = PP, SP, [], check_margins
        self.ok = True

    ids = staticmethod(lambda o: o["params_pred"][:, 145].round().long().tolist())

    def boundary(self, outputs, ratio, ptype="left", torlerance=0.05):
        x = outputs["cam"][:, 2]
        lim = (1 - ratio + torlerance) if ptype == "left" else (ratio - 1 - torlerance)
        if self.check and len(x) and (x - lim).abs().min().item() < MARGIN_X:
            self.ok = False
        before = self.ids(outputs)
        self.SP._orig_exclude(outputs, ratio, ptype=ptype, torlerance=torlerance)
        self.calls.append(("boundary_" + ptype, before, self.ids(outputs)))

    def suppress(self, outputs, img_shape, thresh=16, conf_based=False):
        n = len(outputs["pj2d"])
        if self.check and n > 1:
            pj = outputs["pj2d"]
            d = torch.norm(pj.unsqueeze(1) - pj.unsqueeze(0), p=2, dim=-1).mean(-1)
            sc = outputs["cam"][:, 0] * 2
            dn = d / torch.max(sc.unsqueeze(1).expand(n, n), sc.unsqueeze(0).expand(n, n))
            thr = thresh * max(img_shape) / 640
            iu = torch.triu_indices(n, n, 1)
            if ((dn[iu[0], iu[1]] - thr).abs() / thr).min().item() < MARGIN_REL:
                self.ok = False
        before = self.ids(outputs)
        out = self.PP.suppressing_redundant_prediction_via_projection(outputs, img_shape, thresh=thresh, conf_based=conf_based)
        self.calls.append(("nms", before, self.ids(out)))
        return out

    def outlier(self, outputs, relative_scale_thresh=3, scale_thresh=0.25):
        n = len(outputs["cam_trans"])
        if self.check and n >= 3:
            t = outputs["cam_trans"]
            d = torch.sort(torch.norm(t.unsqueeze(1) - t.unsqueeze(0), p=2, dim=-1)).values[:, 1:-1].mean(1)
            rel = d / ((d.sum() - d) / (n - 1))
            small = outputs["cam"][:, 0] < scale_thresh
            if small.any() and ((rel[small] - relative_scale_thresh).abs() / relative_scale_thresh).min().item() < MARGIN_REL:
                self.ok = False
        before = self.ids(outputs)
        out = self.PP.remove_outlier(outputs, relative_scale_thresh=relative_scale_thresh, scale_thresh=scale_thresh)
        self.calls.append(("outlier", before, self.ids(out)))
        return out


def reference_methods(rec, PP, U):
    """Compile BEV.process_long_image and BEV.single_image_forward from the reference's bev/main.py."""
    path = os.path.join(REF, "bev", "main.py")
    tree = ast.parse(open(path).read(), path)
    cls = next(n for n in tree.body if isinstance(n, ast.ClassDef) and n.name == "BEV")
    fns = [n for n in cls.body if isinstance(n, ast.FunctionDef) and n.name in ("process_long_image", "single_image_forward")]
    assert len(fns) == 2
    g = {"__package__": "bev", "__name__": "bev.main", "torch": torch, "np": np, "img_preprocess": U.img_preprocess,
         "pack_params_dict": PP.pack_params_dict, "denormalize_cam_params_to_trans": PP.denormalize_cam_params_to_trans,
         "body_mesh_projection2image": PP.body_mesh_projection2image,
         "suppressing_redundant_prediction_via_projection": rec.suppress, "remove_outlier": rec.outlier}
    exec(compile(ast.Module(body=fns, type_ignores=[]), path, "exec"), g)
    return g["process_long_image"], g["single_image_forward"]


def stub_self(parser, **kw):
    settings = types.SimpleNamespace(overlap_ratio=0.8, nms_thresh=20, relative_scale_thresh=1.6, center_thresh=0.08,
                                     render_mesh=False, show_patch_results=False, renderer="sim3dr")
    return types.SimpleNamespace(settings=settings, smpl_parser=parser, tdevice=torch.device("cpu"),
                                 result_keys=["smpl_thetas", "smpl_betas", "cam", "cam_trans", "params_pred", "center_confs",
                                              "pred_batch_ids"], **kw)


def post_persons(SP, PP, boxes, pad):
    """Synthetic per-crop outputs of the 256x512 image: one filler per crop plus planted cases (see module docstring)."""
    rs = np.random.RandomState(21)
    k = len(boxes)
    P = []                                         # crop, s, y, x, conf, pose_of (index of a person to copy pose from)

    def add(crop, s, y, x, conf=None, pose_of=None):
        P.append([crop, s, y, x, conf, pose_of])
        return len(P) - 1
    for c in range(k):
        add(c, rs.uniform(1.05, 1.3), -0.1 + 0.02 * (c % 5), 0.0)
    add(0, 1.1, 0.4, 0.8)                          # right part of crop 0 -> left trim
    add(1, 1.1, 0.4, -0.85)                        # left part of crop 1: never trimmed (loop starts at crop 1)
    add(2, 1.1, 0.4, -0.85)                        # left part of crop 2 -> right trim
    f = add(3, 1.1, 0.45, 0.35, conf=0.55)         # duplicates with equal confidence: the later one goes
    add(3, 1.1, 0.45, 0.352, conf=0.55, pose_of=f)
    h_ = add(4, 1.15, -0.45, 0.3, conf=0.31)       # duplicates, the first has the lower confidence: the first goes
    add(4, 1.15, -0.45, 0.301, conf=0.61, pose_of=h_)
    add(5, 1.1, 0.45, -0.35); add(5, 1.2, -0.45, 0.35)
    add(5, 0.1, 0.5, 0.4)                          # far away and small -> per-crop outlier
    p7 = add(7, 1.1, -0.45, 0.35, conf=0.72)       # the same person in crops 7 and 8 -> merged suppression
    p8 = add(8, None, -0.45, None, conf=0.52, pose_of=p7)
    add(10, 0.1, 0.45, 0.3)                        # alone with a filler in its crop, far away -> merged outlier
    n = len(P)
    betas = rs.normal(0, 0.5, (n, 11)).astype(np.float32)
    betas[:, 10] = rs.uniform(0, 0.7, n)
    betas[[2, 9], 10] = 0.9                        # two babies (SMIL)
    thetas = rs.normal(0, 0.25, (n, 72)).astype(np.float32)
    thetas[:, 66:] = 0
    conf = rs.uniform(0.2, 0.99, n).astype(np.float32)
    for i, p in enumerate(P):
        if p[4] is not None:
            conf[i] = p[4]
        if p[5] is not None:
            betas[i], thetas[i] = betas[p[5]], thetas[p[5]]
    # crop 8's copy of the crop-7 person: the same full-image cam (split2process.py:48-58 inverted)
    sc = lambda c: max(int(boxes[c, 1]) - int(boxes[c, 0]), H) / max(H, W)
    sh = lambda c: ((int(boxes[c, 0]) - pad) + (int(boxes[c, 1]) - pad)) / 2 / (W / 2) - 1
    s7, x7 = P[p7][1], P[p7][3]
    P[p8][1] = s7 * sc(7) / sc(8)
    P[p8][3] = ((x7 * sc(7) + sh(7)) - sh(8)) / sc(8)
    cam = np.array([[p[1], p[2], p[3]] for p in P], np.float32)
    params = rs.normal(0, 1, (n, 146)).astype(np.float32)
    params[:, :3] = cam
    params[:, 145] = np.arange(n)                  # person id (read back by the recorder)
    crop_of = np.array([p[0] for p in P], np.int64)
    return crop_of, cam, conf, betas, thetas, params


def post_fixture(PP, SP, U, parser):
    h, w = H, W
    pimg, pad_info, pad = SP.padding_image_overlap(np.zeros((h, w, 3), np.uint8), overlap_ratio=0.8)
    boxes = SP.get_image_split_plan(pimg, overlap_ratio=0.8)
    crop_of, cam, conf, betas, thetas, params = post_persons(SP, PP, boxes, pad)
    rec = Recorder(PP, SP, check_margins=True)
    SP._orig_exclude = SP.exclude_boudary_subjects
    SP.exclude_boudary_subjects = rec.boundary
    process_long_image, _ = reference_methods(rec, PP, U)
    counter = iter(range(len(boxes)))

    def single_image_forward(image):
        c = next(counter)
        l, r, t, b = boxes[c]
        assert image.shape[:2] == (b - t, r - l)
        sel = np.where(crop_of == c)[0]
        out = {"cam": torch.from_numpy(cam[sel]), "center_confs": torch.from_numpy(conf[sel]),
               "smpl_betas": torch.from_numpy(betas[sel]), "smpl_thetas": torch.from_numpy(thetas[sel]),
               "params_pred": torch.from_numpy(params[sel]), "pred_batch_ids": torch.zeros(len(sel), dtype=torch.int64)}
        out["cam_trans"] = PP.denormalize_cam_params_to_trans(out["cam"])
        return out, None
    with torch.no_grad():
        out = process_long_image(stub_self(parser, single_image_forward=single_image_forward), np.zeros((h, w, 3), np.uint8))
    SP.exclude_boudary_subjects = SP._orig_exclude
    assert rec.ok, "a planted decision is too close to its threshold"
    calls = rec.calls
    k = len(boxes)
    # call order: left trims (crops 0..K-2), right trims (crops 2..K-1), per-crop (nms, outlier) x K, merged nms, outlier
    fired = {name: sum(len(b_) - len(a_) for nm, b_, a_ in calls if nm == name) for name in ("boundary_left", "boundary_right")}
    per_crop = [c for c in calls if c[0] in ("nms", "outlier")]
    assert len(per_crop) == 2 * k + 2
    crop_nms = sum(len(b_) - len(a_) for nm, b_, a_ in per_crop[:2 * k:2])
    crop_out = sum(len(b_) - len(a_) for nm, b_, a_ in per_crop[1:2 * k:2])
    m_nms = len(per_crop[2 * k][1]) - len(per_crop[2 * k][2])
    m_out = len(per_crop[2 * k + 1][1]) - len(per_crop[2 * k + 1][2])
    print("removed: left", fired["boundary_left"], "right", fired["boundary_right"], "crop nms", crop_nms, "crop outlier", crop_out,
          "merged nms", m_nms, "merged outlier", m_out)
    assert min(fired.values()) >= 1 and crop_nms >= 2 and crop_out >= 1 and m_nms >= 1 and m_out >= 1
    n = len(cam)
    alive = lambda lists: np.isin(np.arange(n), sorted(set(sum(lists, []))))
    rs = np.random.RandomState(5)
    vsel = rs.choice(6890, 256, replace=False)
    # plan-only records
    plans = []
    for hh, ww in PLAN_SIZES:
        pi, info, pl = SP.padding_image_overlap(np.zeros((hh, ww, 3), np.uint8), overlap_ratio=0.8)
        bx = SP.get_image_split_plan(pi, overlap_ratio=0.8)
        plans.append((pl, bx, info.numpy()))
    np.savez_compressed(
        os.path.join(HERE, "bev_long_post.npz"), h=h, w=w, pad_length=pad, boxes=boxes, pad_info=pad_info.numpy(),
        crop_of=crop_of, cam=cam, conf=conf, betas=betas, thetas=thetas, params_pred=params,
        alive_boundary=alive([c[1] for c in per_crop[:2 * k:2]]), alive_nms=alive([c[2] for c in per_crop[:2 * k:2]]),
        alive_outlier=alive([c[2] for c in per_crop[1:2 * k:2]]), merged_in=np.array(per_crop[2 * k][1]),
        merged_nms=np.array(per_crop[2 * k][2]), final_ids=np.array(per_crop[2 * k + 1][2]),
        out_cam=out["cam"].numpy(), out_cam_trans=out["cam_trans"].numpy(), out_pj2d_org=out["pj2d_org"].numpy(),
        out_joints=out["joints"].numpy(), vsel=vsel, out_verts_sel=out["verts"][:, vsel].numpy(),
        out_conf=out["center_confs"].numpy(), out_thetas=out["smpl_thetas"].numpy(), out_betas=out["smpl_betas"].numpy(),
        out_params_pred=out["params_pred"].numpy(), out_batch_ids=out["pred_batch_ids"].numpy(),
        plan_sizes=np.array(PLAN_SIZES), plan_pad=np.array([p[0] for p in plans]),
        plan_counts=np.array([len(p[1]) for p in plans]), plan_boxes=np.concatenate([p[1] for p in plans]),
        plan_info=np.stack([p[2] for p in plans]))


class PlantedModel:
    """BEVv1.forward (bev/model.py:233-250) with each crop's 3-D centre map replaced by a planted one."""

    def __init__(self, model, vols):
        self.m, self.vols, self.i, self.cache = model, vols, 0, {}

    def __call__(self, x):
        m, i = self.m, self.i
        self.i += 1
        if i not in self.cache:
            feat = m.backbone(x)
            _, cam3d, _ = m.coarse2fine_localization(feat)
            self.cache[i] = (cam3d, m.param_head(feat))
        cam3d, fv = self.cache[i]
        bi, czyx, conf = m.centermap_parser.parse_3dcentermap(torch.from_numpy(self.vols[i:i + 1]))
        if len(bi) == 0:
            return None
        cams = cam3d[bi, :, czyx[:, 0], czyx[:, 1], czyx[:, 2]]
        params, cam_czyx = m.mesh_parameter_regression(fv, cams, bi)
        return {"params_pred": params.float(), "cam_czyx": cam_czyx.float(), "pred_batch_ids": bi, "pred_czyxs": czyx,
                "center_confs": conf}


def model_fixture(PP, SP, U, parser):
    import cv2
    import importlib
    from romp_b200 import synth
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import bev_long_oracle as L
    cv2.ipp.setUseIPP(False)
    M = importlib.import_module("bev.model")
    tt = lambda d: {k: torch.from_numpy(np.asarray(v)) for k, v in d.items()}
    model = M.BEVv1(center_thresh=0.08).eval()
    model.load_state_dict(tt(synth.bev_damp_cam_offsets(synth.bev_state_dict(0))), strict=False)
    image_seed = 17
    image = L.long_image(H, W, image_seed)
    k = len(L.long_image_plan(H, W, 0.8)[1])
    cache = {}
    for vol_seed in range(100):
        vols = L.planted_volumes(k, vol_seed)
        pm = PlantedModel(model, vols)
        pm.cache = cache
        rec = Recorder(PP, SP, check_margins=True)
        SP._orig_exclude = SP.exclude_boudary_subjects
        SP.exclude_boudary_subjects = rec.boundary
        process_long_image, single_image_forward = reference_methods(rec, PP, U)
        me = stub_self(parser, model=pm)
        me.single_image_forward = functools.partial(single_image_forward, me)
        # the reference's filters read person ids from params_pred[:, 145]; keep a copy of the real column per person
        with torch.no_grad():
            try:
                rec.ids = lambda o: o["center_confs"].tolist()
                out = process_long_image(me, image)
            finally:
                SP.exclude_boudary_subjects = SP._orig_exclude
        print("volume seed", vol_seed, "margins ok" if rec.ok else "margin violated", "persons", len(out["cam"]))
        if rec.ok:
            break
    assert rec.ok
    rs = np.random.RandomState(6)
    vsel = rs.choice(6890, 256, replace=False)
    np.savez_compressed(
        os.path.join(HERE, "bev_long_model.npz"), h=H, w=W, image_seed=image_seed, vol_seed=vol_seed, vsel=vsel,
        cam=out["cam"].numpy(), cam_trans=out["cam_trans"].numpy(), center_confs=out["center_confs"].numpy(),
        params_pred=out["params_pred"].numpy(), smpl_thetas=out["smpl_thetas"].numpy(), smpl_betas=out["smpl_betas"].numpy(),
        verts_sel=out["verts"][:, vsel].numpy(), joints=out["joints"].numpy(), pj2d_org=out["pj2d_org"].numpy(),
        pred_batch_ids=out["pred_batch_ids"].numpy(), keys=np.array(sorted(out.keys())))


def main():
    import importlib
    from romp_b200 import synth
    ref = load_reference()
    PP = importlib.import_module("bev.post_parser")
    SP = importlib.import_module("bev.split2process")
    torch.set_num_threads(os.cpu_count())
    tt = lambda d: {k: torch.from_numpy(np.asarray(v)) for k, v in d.items()}
    with tempfile.TemporaryDirectory() as d:
        torch.save(tt(synth.smpl_pack(0, num_betas=11)), os.path.join(d, "a.pth"))
        torch.save(tt(synth.smpl_pack(1)), os.path.join(d, "s.pth"))
        parser = PP.SMPLA_parser(os.path.join(d, "a.pth"), os.path.join(d, "s.pth"))
    post_fixture(PP, SP, ref["romp.utils"], parser)
    if "post" not in sys.argv[1:]:
        model_fixture(PP, SP, ref["romp.utils"], parser)
    for f in sorted(os.listdir(HERE)):
        if f.startswith("bev_long"):
            print(f, os.path.getsize(os.path.join(HERE, f)))


if __name__ == "__main__":
    main()
