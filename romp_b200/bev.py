"""Drop-in call surface of ``simple_romp``'s BEV (bev/main.py) on the GPU hot path.

``bev_settings`` mirrors bev/main.py:27-87 (same flags and defaults, including the quirk that ``crowd`` defaults to
True and therefore overrides the thresholds with ``long_conf_dict``), ``BEV(settings)(image_bgr) -> dict | None``
mirrors bev/main.py:91-258: normal images run as one 512x512 frame, and in crowd mode images at least twice as wide as
high run through ``process_long_image`` (the reference's overlapping crops, batched through the model, with the per-crop
and merged filters on the device).  ``forward_batch`` is the batched entry point for normal frames, ``forward_images`` the
batched ``forward`` on raw images of different sizes (each frame with its own geometry).
Per-frame semantics of the two post filters (bev/post_parser.py:167-222) are preserved by applying them per
``pred_batch_ids`` group on the device.  Python only allocates buffers and sequences library calls.
"""
from __future__ import annotations

import argparse
import ctypes as C
import os
import os.path as osp
import sys

import numpy as np
import torch

from . import _lib, graph
from ._lib import BF16, F32, U8
from .main import MAX_PERSON, SMPLParser, _ptr, img_preprocess
from .staging import RawStager, after_producers, frame_buffer, frame_offsets, image_tensor, preprocess_bgr_batch, split_by_frame

conf_dict = {1: [0.25, 20, 2], 2: [0.1, 20, 1.6]}                    # bev/main.py:24-25
long_conf_dict = {1: [0.12, 20, 1.5, 0.46], 2: [0.08, 20, 1.6, 0.8]}
model_dict = {1: "BEV_ft_agora.pth", 2: "BEV.pth"}
N_PARAMS = 146                                                       # 3 cam + 22*6 + 11 betas, bev/model.py:116
TRACKER_MAX_TRACKS = 128                                             # live tracks (tracked + lost) of the video mode
MAX_SIGNALS = 4                                                      # filter sets of the video mode, the oldest evicted


def bev_settings(input_args=sys.argv[1:]):
    """Same flags/defaults as bev/main.py:27-87; no downloads, no prints."""
    model_id = 2
    home = osp.join(osp.expanduser("~"), ".romp")
    p = argparse.ArgumentParser(description="BEV (GPU-native hot path)")
    p.add_argument("-m", "--mode", type=str, default="image")
    p.add_argument("--model_id", type=int, default=2)
    p.add_argument("-i", "--input", type=str, default=None)
    p.add_argument("-o", "--save_path", type=str, default=osp.join(osp.expanduser("~"), "BEV_results"))
    p.add_argument("--crowd", action="store_false")
    p.add_argument("--GPU", type=int, default=0)
    p.add_argument("--overlap_ratio", type=float, default=long_conf_dict[model_id][3])
    p.add_argument("--center_thresh", type=float, default=conf_dict[model_id][0])
    p.add_argument("--nms_thresh", type=float, default=conf_dict[model_id][1])
    p.add_argument("--relative_scale_thresh", type=float, default=conf_dict[model_id][2])
    p.add_argument("--show_largest", action="store_true")
    p.add_argument("--show_patch_results", action="store_true")
    p.add_argument("--calc_smpl", action="store_false")
    p.add_argument("--renderer", type=str, default="sim3dr")
    p.add_argument("--render_mesh", action="store_false")
    p.add_argument("--show", action="store_true")
    p.add_argument("--show_items", type=str, default="mesh,mesh_bird_view")
    p.add_argument("--save_video", action="store_true")
    p.add_argument("--frame_rate", type=int, default=24)
    p.add_argument("--smpl_path", type=str, default=osp.join(home, "SMPLA_NEUTRAL.pth"))
    p.add_argument("--smil_path", type=str, default=osp.join(home, "smil_packed_info.pth"))
    p.add_argument("--model_path", type=str, default=osp.join(home, model_dict[model_id]))
    p.add_argument("-t", "--temporal_optimize", action="store_true")
    p.add_argument("-sc", "--smooth_coeff", type=float, default=3.0)
    p.add_argument("--webcam_id", type=int, default=0)
    p.add_argument("--precision", type=str, default="bf16", choices=["bf16", "tf32", "fp32"])
    p.add_argument("--max_batch", type=int, default=32)
    args = p.parse_args(input_args)
    if args.model_id != 2:                                            # bev/main.py:59-63
        args.model_path = osp.join(home, model_dict[args.model_id])
        args.center_thresh, args.nms_thresh = conf_dict[args.model_id][0], conf_dict[args.model_id][1]
        args.relative_scale_thresh = conf_dict[model_id][2]
    if args.crowd:                                                    # :81-85 (crowd defaults to True)
        args.center_thresh, args.nms_thresh = long_conf_dict[args.model_id][0], long_conf_dict[args.model_id][1]
        args.relative_scale_thresh, args.overlap_ratio = long_conf_dict[model_id][2], long_conf_dict[args.model_id][3]
    return args


def long_image_plan(h, w, overlap_ratio):
    """padding_image_overlap + get_image_split_plan (bev/split2process.py:6-39) for an h x w image.

    Returns (pad_length, boxes int32 [K,4] of [left, right, top, bottom] in the horizontally zero-padded image of width
    w + 2*pad_length, pad_info6 of the full image).  Same float arithmetic and int32 truncation as the reference,
    including its last box: left = W - h but the previous box's right, so it is narrower than h."""
    pad_length = int(h * overlap_ratio)
    W = w + 2 * pad_length
    k = int(np.ceil((W / h - 1) / (1 - overlap_ratio))) + 1
    step = (1 - overlap_ratio) * h
    boxes, right = [], None
    for i in range(k):
        if i == k - 1:
            left = W - h
        else:
            left = step * i
            right = left + h
        boxes.append([left, right, 0, h])
    top = (w - h) // 2
    return pad_length, np.array(boxes).astype(np.int32), np.array([top, w - top, 0, w, h, w], np.float32)


def long_image_crop_table(boxes, pad_length, h, w, nms_thresh):
    """Per-crop constants of the long-image stages (fp32 [K,6], see b200romp_bev_crop_post): boundary limits
    (bev/main.py:209-226), projection size and suppression pixels (:216-217,231), cam scale and x shift
    (split2process.py:48-58; float64 on the host, applied to fp32 like the reference's in-place ops)."""
    k = len(boxes)
    tab = np.zeros((k, 6), np.float64)
    ratio = [(int(boxes[i, 1]) - int(boxes[i + 1, 0])) / h / 2 for i in range(k - 1)]
    for i, (l, r, t, b) in enumerate(boxes.tolist()):
        side = max(b - t, r - l)
        tab[i, 0] = 1 - ratio[i] if i < k - 1 else np.inf
        tab[i, 1] = ratio[i - 1] - 1 if i >= 2 else -np.inf
        tab[i, 2] = side
        tab[i, 3] = nms_thresh * side / 640
        tab[i, 4] = max(r - l, b - t) / max(h, w)
        tab[i, 5] = ((l - pad_length) + (r - pad_length)) / 2 / (w / 2) - 1
    return tab.astype(np.float32)


class BEV(torch.nn.Module):
    """``BEV(settings)(image_bgr)`` - the contract of simple_romp/bev/main.py:91-258 (normal and crowd-mode images)."""

    result_keys = ["smpl_thetas", "smpl_betas", "cam", "cam_trans", "params_pred", "center_confs", "pred_batch_ids"]   # :115

    def __init__(self, settings, state_dict=None, smpla_pack=None, smil_pack=None):
        super().__init__()
        self.settings = s = settings
        if not torch.cuda.is_available() or s.GPU < 0:
            raise RuntimeError("romp_b200.BEV needs a CUDA device (H100, sm_90a); there is no CPU fallback")
        if getattr(s, "show", False):
            raise NotImplementedError("display (--show) is outside the GPU hot path (SURVEY.md section 2)")
        self.temporal = bool(getattr(s, "temporal_optimize", False))
        self.show_largest = self.temporal and bool(getattr(s, "show_largest", False))
        # NB the reference renders by default (render_mesh is store_false, bev/main.py:44); rendering is out of scope and
        # simply not performed here.
        self.lib = _lib.load()
        self.device_index = int(s.GPU)
        self.tdevice = torch.device("cuda", self.device_index)
        torch.cuda.set_device(self.tdevice)
        self.precision = getattr(s, "precision", "bf16")
        self._frames = {}                              # frame buffers by (dtype, B)
        self.max_batch = B = int(getattr(s, "max_batch", 32))
        if state_dict is None:
            state_dict = torch.load(s.model_path, map_location="cpu")          # bev/main.py:101 (strict=False)
        self._sd = state_dict
        self._nets = {}
        self.stream = torch.cuda.Stream(device=self.tdevice)
        w = graph.bev_weights(state_dict)
        self._w_keep = w
        fp = C.POINTER(C.c_float)
        bw = _lib.BevWeights(*[w[k].ctypes.data_as(fp) for k in ("center_ref", "cam_ref", "coordmap", "anchors", "embed",
                                                                   "w0", "b0", "w1", "b1", "w2", "b2")])
        self.h = self.lib.b200romp_bev_create(self.device_index, C.byref(bw))
        if not self.h:
            raise RuntimeError("b200romp_bev_create: " + self.lib.b200romp_last_error().decode())
        self.calc_smpl = bool(s.calc_smpl)
        if self.calc_smpl:
            if smpla_pack is None:
                smpla_pack = torch.load(s.smpl_path, map_location="cpu")
            if smil_pack is None:
                smil_pack = torch.load(s.smil_path, map_location="cpu")
            self.smpla = SMPLParser(smpla_pack, self.device_index, n_betas=11, shape_key="smpla_shapedirs")   # post_parser.py:259
            self.smil = SMPLParser(smil_pack, self.device_index, n_betas=10)                                     # :258
        self._alloc(B)
        if self.temporal:
            self._alloc_temporal(B)

    def _net(self, in_dtype):
        if in_dtype not in self._nets:
            self._nets[in_dtype] = graph.build_bev(self._sd, self.device_index, self.precision, in_dtype, self.max_batch)
        return self._nets[in_dtype]

    def _alloc(self, B):
        dev, cap = self.tdevice, B * MAX_PERSON
        self.cap = cap
        act = torch.bfloat16 if self.precision == "bf16" else torch.float32
        self.act_code = BF16 if self.precision == "bf16" else F32
        z = lambda *shape, dtype=torch.float32: torch.zeros(*shape, dtype=dtype, device=dev)
        i64, i32 = torch.int64, torch.int32
        self.buf = dict(
            maps_fv=z(B, 4, 128, 128), fv_feats=z(B, 128, 128, 128, dtype=act), img_feats=z(B, 128, 128, graph.bev_feats_channels(self.precision), dtype=act),
            bv_in=z(B, 1, 128, 2560, dtype=act), bv_out=z(B, 1, 128, 128, dtype=act),
            c3d_tmp=z(B, 64, 128, 128), center3d=z(B, 64, 128, 128),
            parse_ws=torch.zeros(int(self.lib.b200romp_bev_parse_workspace_bytes(B)), dtype=torch.uint8, device=dev),
            count=z(1, dtype=i32), batch_ids=z(cap, dtype=i64), czyx=z(cap, 3, dtype=i64), conf=z(cap),
            params_pred=z(cap, N_PARAMS), cam_czyx=z(cap, 3, dtype=i64), cam=z(cap, 3), thetas=z(cap, 72), betas=z(cap, 11),
            cam_trans=z(cap, 3), pj2d_org=z(cap, 71, 2), keep=z(cap, dtype=i32), sel=z(cap, dtype=i32), count2=z(1, dtype=i32),
        )
        if self.calc_smpl:
            self.buf.update(verts=z(cap, 6890, 3), joints=z(cap, 71, 3), verts_smil=z(cap, 6890, 3), joints_smil=z(cap, 71, 3),
                            smpl_ws=z(cap, self.smpla.ws_floats))
        # compacted outputs (after the per-frame post filters)
        self.out = {k: torch.zeros_like(self.buf[k]) for k in ("batch_ids", "conf", "params_pred", "cam", "thetas", "betas",
                                                               "cam_trans", "pj2d_org")}
        if self.calc_smpl:
            self.out.update(verts=torch.zeros_like(self.buf["verts"]), joints=torch.zeros_like(self.buf["joints"]))
        self.count_host = torch.zeros(2, dtype=torch.int32).pin_memory()
        self.pad_table = z(B, 6)                       # per-frame pad info of forward_images / forward_batch([B,6] offsets)
        self.raw = RawStager(dev)                       # raw image staging of forward_images

    def _alloc_temporal(self, B):
        """The video mode (bev/main.py:109-121,260-287): one tracker per instance (shared by every signal_ID), the
        filter sets of MAX_SIGNALS signals, and row buffers for up to 2 x 64 rows per frame."""
        dev, R = self.tdevice, 2 * B * MAX_PERSON
        self.trk = self.lib.b200romp_bev_tracker_create(self.device_index, TRACKER_MAX_TRACKS, MAX_SIGNALS)
        if not self.trk:
            raise RuntimeError("b200romp_bev_tracker_create: " + self.lib.b200romp_last_error().decode())
        self.signals = {}                              # signal_ID -> filter set, oldest first (ROMP's TemporalState)
        z = lambda *shape, dtype=torch.float32: torch.zeros(*shape, dtype=dtype, device=dev)
        i64, i32 = torch.int64, torch.int32
        self.tbuf = dict(count=z(1, dtype=i32), batch_ids=z(R, dtype=i64), track_ids=z(R, dtype=i32), det=z(R, dtype=i32),
                         thetas=z(R, 72), betas=z(R, 11), cam=z(R, 3), cam_trans=z(R, 3), params_pred=z(R, N_PARAMS), conf=z(R),
                         status=z(2 + B, dtype=i32), sig=z(B, dtype=i32), pj2d_org=z(R, 71, 2), keep=z(R, dtype=i32),
                         sel=z(R, dtype=i32), count2=z(1, dtype=i32))
        if self.calc_smpl:
            self.tbuf.update(verts=z(R, 6890, 3), joints=z(R, 71, 3), verts_smil=z(R, 6890, 3), joints_smil=z(R, 71, 3),
                             smpl_ws=z(R, self.smpla.ws_floats))
        self.tout = {k: torch.zeros_like(self.tbuf[k]) for k in ("batch_ids", "track_ids", "conf", "params_pred", "cam", "thetas",
                                                                "betas", "cam_trans", "pj2d_org")}
        if self.calc_smpl:
            self.tout.update(verts=torch.zeros_like(self.tbuf["verts"]), joints=torch.zeros_like(self.tbuf["joints"]))
        # the batch's one read-back: detected, rows, kept rows, then the kernel's status, frame_id and rows per frame
        self.tsync_host = torch.zeros(5 + B, dtype=torch.int32).pin_memory()
        self.frame_id = 0                              # tracker frames so far (frames with a detection)
        self.tsig_host = torch.zeros(B, dtype=torch.int32).pin_memory()

    def _signal_slots(self, signal_IDs):
        """filter set of every frame's signal_ID; a new signal beyond MAX_SIGNALS evicts the oldest one (its filters are
        reset on the stream, before the batch's kernel)."""
        if len(set(signal_IDs)) > MAX_SIGNALS:
            raise ValueError(f"BEV video mode: at most {MAX_SIGNALS} distinct signal_IDs per batch (their filter sets are "
                             "used by one kernel); split the batch")
        slots = []
        batch = set(signal_IDs)
        for sid in signal_IDs:
            if sid not in self.signals:
                if len(self.signals) >= MAX_SIGNALS:                       # the oldest signal not used by this batch
                    self.signals.pop(next(k for k in self.signals if k not in batch))
                used = set(self.signals.values())
                slot = next(k for k in range(MAX_SIGNALS) if k not in used)
                _lib.check(self.lib.b200romp_bev_tracker_reset(self.trk, slot, C.c_void_p(self.stream.cuda_stream)), "tracker_reset")
                self.signals[sid] = slot
            slots.append(self.signals[sid])
        return slots

    def reset_temporal(self):
        """Forget every track, id and filter (a new video); ids start again from 1."""
        if not self.temporal:
            raise RuntimeError("reset_temporal: this BEV instance was built without -t/--temporal_optimize")
        _lib.check(self.lib.b200romp_bev_tracker_reset(self.trk, -1, C.c_void_p(self.stream.cuda_stream)), "tracker_reset")
        self.signals = {}

    @torch.no_grad()
    def run_temporal(self, B, signal_IDs):
        """BEV.temporal_optimization (bev/main.py:165-169,260-287) of the batch's frames in order: one kernel
        (b200romp_bev_track_step) between the regressor and SMPL-A, writing the smoothed rows to ``self.tbuf``."""
        b, t = self.buf, self.tbuf
        slots = self._signal_slots(signal_IDs)
        self.tsig_host[:B].copy_(torch.tensor(slots, dtype=torch.int32))
        t["sig"][:B].copy_(self.tsig_host[:B], non_blocking=True)
        R = 2 * B * MAX_PERSON
        _lib.check(self.lib.b200romp_bev_track_step(
            self.trk, B, B * MAX_PERSON, _ptr(b["count"]), _ptr(b["batch_ids"]), _ptr(b["conf"]), _ptr(b["cam"]), _ptr(b["cam_trans"]),
            _ptr(b["thetas"]), _ptr(b["betas"]), _ptr(b["params_pred"]), _ptr(t["sig"]), int(self.show_largest),
            float(self.settings.smooth_coeff), R, _ptr(t["count"]), _ptr(t["batch_ids"]), _ptr(t["track_ids"]), _ptr(t["det"]),
            _ptr(t["thetas"]), _ptr(t["betas"]), _ptr(t["cam"]), _ptr(t["cam_trans"]), _ptr(t["params_pred"]), _ptr(t["conf"]),
            _ptr(t["status"]), C.c_void_p(self.stream.cuda_stream)), "bev_track_step")

    @torch.no_grad()
    def run_post_temporal(self, B, offsets, img_max_side=512.0):
        """run_post on the tracker's rows (up to 2 x 64 per frame)."""
        self.run_post(B, offsets, img_max_side, self.tbuf, self.tout, 2 * B * MAX_PERSON, self.tbuf["count"])

    def _collect_temporal(self, B, to_numpy):
        """(batch result dict, rows per frame) after the host sync; raises on a full track table."""
        h, t = self.tsync_host, self.tbuf
        with torch.cuda.stream(self.stream):
            h[0:1].copy_(self.buf["count"], non_blocking=True)
            h[1:2].copy_(t["count"], non_blocking=True)
            h[2:3].copy_(t["count2"], non_blocking=True)
            h[3:5 + B].copy_(t["status"][:2 + B], non_blocking=True)
        self.stream.synchronize()
        n_det, n_rows, n_kept, status = int(h[0]), int(h[1]), int(h[2]), int(h[3])
        self.frame_id = int(h[4])
        if status:
            raise RuntimeError("BEV video mode: " + (f"more than {TRACKER_MAX_TRACKS} live tracks" if status == 1 else "too many rows")
                               + "; call reset_temporal() before the next frame")
        src, n = (self.tout, n_kept) if self.calc_smpl else (self.tbuf, n_rows)
        bid = src["batch_ids"][:n]
        out = self._result(src, n, bid, False)
        out["_bid"] = bid
        if not self.show_largest:
            out["track_ids"] = src["track_ids"][:n]
        else:                                           # bev/main.py:262-267: only thetas / betas / cam are cut to one row
            out.update(params_pred=self.buf["params_pred"][:n_det], center_confs=self.buf["conf"][:n_det],
                       pred_batch_ids=self.buf["batch_ids"][:n_det])
        rows = {b for b in range(B) if int(h[5 + b])}                # frames the tracker gave rows (before the filters)
        if to_numpy:
            with torch.cuda.stream(self.stream):
                out = {k: v.contiguous().cpu().numpy() for k, v in out.items()}
        return out, rows

    def _split_temporal(self, out, B, rows, to_numpy):
        """per-frame dicts of a temporal batch result (None for a frame without rows), pred_batch_ids set to 0."""
        res = []
        for b in range(B):
            if b not in rows:
                res.append(None)
                continue
            r = {}
            for k, v in out.items():
                ids = out["pred_batch_ids"] if (self.show_largest and k in ("params_pred", "center_confs", "pred_batch_ids")) else out["_bid"]
                r[k] = v[ids == b]
            n = len(r["pred_batch_ids"])
            r["pred_batch_ids"] = np.zeros(n, np.int64) if to_numpy else torch.zeros(n, dtype=torch.int64, device=self.tdevice)
            r.pop("_bid")
            res.append(r)
        return res

    # ------------------------------------------------------------------------------------------
    @torch.no_grad()
    def run_model(self, frames_dev, center3d_override=None):
        """BEVv1.forward (bev/model.py:232-250) + pack_params_dict / cam_trans (bev/main.py:128-129); no host sync."""
        B = frames_dev.shape[0]
        assert frames_dev.is_cuda and frames_dev.is_contiguous() and tuple(frames_dev.shape[1:]) == (512, 512, 3)
        assert B <= self.max_batch
        in_dtype = {torch.uint8: U8, torch.float32: F32}[frames_dev.dtype]
        g1, io1, g2, io2 = self._net(in_dtype)
        lib, b, sp, ac = self.lib, self.buf, C.c_void_p(self.stream.cuda_stream), self.act_code
        ck = _lib.check
        ck(lib.b200romp_net_bind(g1.net, io1["frames"], _ptr(frames_dev)))
        ck(lib.b200romp_net_bind(g1.net, io1["maps_fv"], _ptr(b["maps_fv"])))
        ck(lib.b200romp_net_bind(g1.net, io1["fv_feats"], _ptr(b["fv_feats"])))
        ck(lib.b200romp_net_bind(g1.net, io1["img_feats"], _ptr(b["img_feats"])))
        ck(lib.b200romp_net_run(g1.net, B, sp), "net_run(g1)")
        ck(lib.b200romp_bev_bv_input(_ptr(b["maps_fv"]), _ptr(b["img_feats"]), ac, b["img_feats"].shape[-1], B, _ptr(b["bv_in"]), ac, sp),
           "bv_input")
        ck(lib.b200romp_net_bind(g2.net, io2["bv_in"], _ptr(b["bv_in"])))
        ck(lib.b200romp_net_bind(g2.net, io2["bv_out"], _ptr(b["bv_out"])))
        ck(lib.b200romp_net_run(g2.net, B, sp), "net_run(g2)")
        ck(lib.b200romp_bev_center3d(self.h, _ptr(b["maps_fv"]), _ptr(b["bv_out"]), ac, B, _ptr(b["c3d_tmp"]), _ptr(b["center3d"]), sp),
           "center3d")
        c3d = b["center3d"] if center3d_override is None else center3d_override
        ck(lib.b200romp_bev_parse3d(_ptr(c3d), B, float(self.settings.center_thresh), self.cap, _ptr(b["count"]), _ptr(b["batch_ids"]),
                                    _ptr(b["czyx"]), _ptr(b["conf"]), _ptr(b["parse_ws"]), sp), "parse3d")
        ck(lib.b200romp_bev_regress(self.h, _ptr(b["maps_fv"]), _ptr(b["bv_out"]), ac, _ptr(b["fv_feats"]), ac, B * MAX_PERSON,
                                    _ptr(b["count"]), _ptr(b["batch_ids"]), _ptr(b["czyx"]), _ptr(b["params_pred"]),
                                    _ptr(b["cam_czyx"]), _ptr(b["cam"]), _ptr(b["thetas"]), _ptr(b["betas"]), _ptr(b["cam_trans"]), sp),
           "regress")

    @torch.no_grad()
    def run_post(self, B, offsets, img_max_side=512.0, b=None, o=None, cap=None, count=None):
        """SMPLA_parser + projection + the two per-frame filters (bev/main.py:172-180), then row compaction.  ``offsets``:
        one pad info for every frame (suppression with ``img_max_side``), or a device [B,6] table with one row per frame
        (each frame projects and suppresses with its own size).  b / o / cap / count: the row buffers (default: the
        regressor's rows)."""
        lib, sp = self.lib, C.c_void_p(self.stream.cuda_stream)
        b = self.buf if b is None else b
        o = self.out if o is None else o
        cap = B * MAX_PERSON if cap is None else cap
        count = b["count"] if count is None else count
        if not self.calc_smpl:
            return
        st = self.stream.cuda_stream
        self.smpla.forward(b["betas"], b["thetas"], cap, count, True, b["smpl_ws"], b["verts"], b["joints"], st)
        self.smil.forward(b["betas"], b["thetas"], cap, count, True, b["smpl_ws"], b["verts_smil"], b["joints_smil"], st)
        args = (_ptr(b["betas"]), _ptr(b["verts_smil"]), _ptr(b["joints_smil"]), _ptr(b["verts"]), _ptr(b["joints"]), _ptr(b["cam"]),
                _ptr(b["cam_trans"]), _ptr(b["batch_ids"]), B, cap, _ptr(count))
        if isinstance(offsets, torch.Tensor) and offsets.dim() == 2:
            _lib.check(lib.b200romp_bev_post_frames(*args, _ptr(offsets), float(self.settings.nms_thresh),
                                                    float(self.settings.relative_scale_thresh), _ptr(b["pj2d_org"]), _ptr(b["keep"]),
                                                    _ptr(b["sel"]), _ptr(b["count2"]), sp), "bev_post_frames")
        else:
            off = (C.c_float * 6)(*[float(v) for v in offsets])
            _lib.check(lib.b200romp_bev_post(*args, off, float(self.settings.nms_thresh), float(self.settings.relative_scale_thresh),
                                             float(img_max_side), _ptr(b["pj2d_org"]), _ptr(b["keep"]), _ptr(b["sel"]),
                                             _ptr(b["count2"]), sp), "bev_post")
        for k, dst in o.items():
            src = b["conf"] if k == "conf" else b[k]
            row = src[0].numel() * src.element_size()
            _lib.check(lib.b200romp_gather_rows(_ptr(src), row, _ptr(b["sel"]), _ptr(b["count2"]), cap, _ptr(dst), sp), "gather_rows")

    def _counts(self, detected, kept):
        """The host sync of a result: (persons detected, persons kept by the filters) from two device counters."""
        with torch.cuda.stream(self.stream):
            self.count_host[0:1].copy_(detected, non_blocking=True)
            self.count_host[1:2].copy_(kept, non_blocking=True)
        self.stream.synchronize()
        return int(self.count_host[0]), int(self.count_host[1])

    def _result(self, src, n, batch_ids, to_numpy):
        """The output dict (result_keys, plus the SMPL outputs) from the first n rows of the buffers ``src``."""
        out = {"smpl_thetas": src["thetas"][:n], "smpl_betas": src["betas"][:n], "cam": src["cam"][:n], "cam_trans": src["cam_trans"][:n],
               "params_pred": src["params_pred"][:n], "center_confs": src["conf"][:n], "pred_batch_ids": batch_ids}
        if self.calc_smpl:
            out.update(verts=src["verts"][:n], joints=src["joints"][:n], pj2d_org=src["pj2d_org"][:n])
        if to_numpy:
            with torch.cuda.stream(self.stream):
                out = {k: v.contiguous().cpu().numpy() for k, v in out.items()}
        return out

    def collect(self, to_numpy=True):
        n_det, n = self._counts(self.buf["count"], self.buf["count2"])
        if n_det == 0:
            return None
        src, n = (self.out, n) if self.calc_smpl else (self.buf, n_det)
        return self._result(src, n, src["batch_ids"][:n], to_numpy)

    @torch.no_grad()
    def forward_batch(self, frames, offsets=None, to_numpy=True, center3d_override=None, img_max_side=512.0, signal_IDs=None):
        """frames [B,512,512,3] padded+resized like img_preprocess.  ``offsets``: one pad info [top,bottom,left,right,h,w]
        for every frame, suppressing with ``img_max_side``; or one row per frame ([B,6], numpy or tensor), each frame then
        suppressing with its own max(h, w) (``img_max_side`` is not used).  With -t the frames are consecutive video
        frames, tracked and smoothed in order (``signal_IDs``: one per frame, default 0); the result adds ``track_ids``."""
        if isinstance(frames, np.ndarray):
            frames = torch.from_numpy(frames)
        B = frames.shape[0]
        after_producers(self.stream, self.tdevice, frames, center3d_override, offsets)
        fd = frame_buffer(self._frames, frames.dtype, B, self.tdevice)
        with torch.cuda.stream(self.stream):
            fd.copy_(frames, non_blocking=True)
            offsets = frame_offsets(offsets, self.pad_table, B)
            self.run_model(fd, center3d_override)
            if self.temporal:
                self.run_temporal(B, [0] * B if signal_IDs is None else list(signal_IDs))
                self.run_post_temporal(B, offsets, img_max_side)
            else:
                self.run_post(B, offsets, img_max_side)
        if self.temporal:
            out, rows = self._collect_temporal(B, to_numpy)
            out.pop("_bid")
            return out if rows else None
        return self.collect(to_numpy)

    @torch.no_grad()
    def forward_images(self, images, to_numpy=True, center3d_override=None, signal_IDs=None):
        """Batched ``forward`` on raw images of any sizes (HxWx3 uint8 BGR: numpy arrays, host or device tensors): a list
        of the same length, element i the result for images[i] (dict or None; nothing is printed for normal images).
        Normal images run in chunks of at most ``max_batch`` through one preprocessing kernel per chunk (the GPU kernel,
        not the host OpenCV resize of ``forward``) and b200romp_bev_post_frames, each frame with its own pad info and
        suppression threshold; element i then equals ``forward_batch`` on image i's GPU-preprocessed frame with its pad
        info and ``img_max_side = max(h, w)``.  In crowd mode images with w/h >= 2 go one by one through
        ``process_long_image``.  center3d_override: optional device [n_normal,64,128,128] for the normal images in order.
        With -t the normal images are consecutive video frames (``signal_IDs``: one per image, default 0), tracked and
        smoothed in list order; wide crowd-mode images are neither tracked nor smoothed (bev/main.py:140-143)."""
        imgs = [image_tensor(x) for x in images]
        res = [None] * len(imgs)
        normal = []
        for i, t in enumerate(imgs):
            if self.settings.crowd and t.shape[1] / t.shape[0] >= 2:
                if getattr(self.settings, "show_patch_results", False):
                    raise NotImplementedError("show_patch_results renders and saves per-crop images; rendering is out of scope")
                res[i] = self.process_long_image(t, to_numpy=to_numpy)
            else:
                normal.append(i)
        if center3d_override is not None:
            assert center3d_override.is_cuda and center3d_override.shape[0] == len(normal)
            after_producers(self.stream, self.tdevice, center3d_override)
        for c0 in range(0, len(normal), self.max_batch):
            idx = normal[c0:c0 + self.max_batch]
            sigs = [0 if signal_IDs is None else signal_IDs[i] for i in idx]
            for i, r in zip(idx, self._forward_chunk([imgs[i] for i in idx], to_numpy,
                                                     None if center3d_override is None else center3d_override[c0:c0 + len(idx)], sigs)):
                res[i] = r
        return res

    def _forward_chunk(self, imgs, to_numpy, center3d_override, signal_IDs=None):
        """One chunk of normal images: staging + one H2D, batched preprocessing, model, per-frame post; one host sync."""
        B = len(imgs)
        # the previous chunk ended in a host sync: the pinned buffer is free, and self.stream is the last reader of both
        offs, total = self.raw.stage(imgs, replace_after=self.stream)
        after_producers(self.stream, self.tdevice, *imgs)
        fd = frame_buffer(self._frames, torch.uint8, B, self.tdevice)
        with torch.cuda.stream(self.stream):
            if total:
                self.raw.upload(total)
            preprocess_bgr_batch(self.lib, imgs, offs, self.raw.dev, fd, self.pad_table, self.stream.cuda_stream)
            self.run_model(fd, center3d_override)
            if self.temporal:
                self.run_temporal(B, signal_IDs)
                self.run_post_temporal(B, self.pad_table[:B])
            else:
                self.run_post(B, self.pad_table[:B])
        if self.temporal:
            out, rows = self._collect_temporal(B, to_numpy)
            return self._split_temporal(out, B, rows, to_numpy)
        out = self.collect(to_numpy)
        if out is None:
            return [None] * B
        n_det = int(self.count_host[0])
        detected = set(self.buf["batch_ids"][:n_det].cpu().tolist())       # frames with a detection (before the filters)
        res = split_by_frame(out, B, to_numpy)
        for i, r in enumerate(res):
            n = len(r["cam"])
            r["pred_batch_ids"] = np.zeros(n, np.int64) if to_numpy else torch.zeros(n, dtype=torch.int64, device=self.tdevice)
        return [r if i in detected else None for i, r in enumerate(res)]      # an undetected frame alone returns None

    def _long_buffers(self, rows):
        """Image-level accumulation rows of the long-image mode (grown on demand, kept for the next image)."""
        lb = getattr(self, "_long", None)
        if lb is not None and lb["cam"].shape[0] >= rows:
            return lb
        dev = self.tdevice
        z = lambda *shape, dtype=torch.float32: torch.zeros(*shape, dtype=dtype, device=dev)
        lb = dict(verts=z(rows, 6890, 3), joints=z(rows, 71, 3), thetas=z(rows, 72), betas=z(rows, 11), params_pred=z(rows, N_PARAMS),
                  conf=z(rows), cam=z(rows, 3), cam_trans=z(rows, 3), pj2d_org=z(rows, 71, 2), removed=z(rows, dtype=torch.int32),
                  sel=z(rows, dtype=torch.int32), count=z(2, dtype=torch.int32), count2=z(1, dtype=torch.int32),
                  ctl=z(2, dtype=torch.int32), cam_full=z(self.cap, 3),
                  ws=torch.zeros(int(self.lib.b200romp_bev_long_merge_workspace_bytes(rows)), dtype=torch.uint8, device=dev))
        lb["out"] = {k: torch.zeros_like(lb[k]) for k in ("verts", "joints", "thetas", "betas", "params_pred", "conf", "cam",
                                                          "cam_trans", "pj2d_org")}
        self._long = lb
        return lb

    @torch.no_grad()
    def process_long_image(self, full_image, center3d_override=None, to_numpy=True):
        """Crowd mode for images at least twice as wide as high, bev/main.py:184-258 (``BEV.forward`` dispatches here).

        The image is zero-padded horizontally on the device and cut into the reference's overlapping crops
        (``long_image_plan``); every crop becomes a 512x512 frame (b200romp_preprocess_bgr on the crop's window of the
        padded image), the crops run through the model in chunks of at most ``max_batch`` frames, each chunk's
        persons go through the per-crop filters and are appended to image-level rows (b200romp_bev_crop_post), and
        the merged filters run on those rows (b200romp_bev_long_merge).  One host sync per image.
        center3d_override: optional device [K,64,128,128] replacing the crops' 3-D centre maps (tests, measurement)."""
        if not self.calc_smpl:
            raise ValueError("the long-image mode needs SMPL (bev/main.py:203): calc_smpl must be on for images with w/h >= 2")
        img = image_tensor(full_image)
        s = self.settings
        h, w = int(img.shape[0]), int(img.shape[1])
        pad_length, boxes, pad_info = long_image_plan(h, w, s.overlap_ratio)
        K, B = len(boxes), self.max_batch
        if center3d_override is not None:
            assert center3d_override.is_cuda and tuple(center3d_override.shape) == (K, 64, 128, 128)
            after_producers(self.stream, self.tdevice, center3d_override)
        lb = self._long_buffers(K * MAX_PERSON)
        tab = torch.from_numpy(long_image_crop_table(boxes, pad_length, h, w, float(s.nms_thresh))).pin_memory()
        frames = frame_buffer(self._frames, torch.uint8, B, self.tdevice)
        with torch.cuda.stream(self.stream):
            padded = self.pad_long_image(img, pad_length)
            tab_dev = tab.to(self.tdevice, non_blocking=True)
            lb["count"].zero_()
            for c0 in range(0, K, B):
                nb = min(B, K - c0)
                self.crop_frames(padded, boxes[c0:c0 + nb], frames)                         # main.py:197-199 + img_preprocess
                self.run_model(frames[:nb], None if center3d_override is None else center3d_override[c0:c0 + nb])
                self.crop_post(nb, c0, tab_dev)
            self.long_merge(pad_info, w)
        return self._collect_long(to_numpy)

    def pad_long_image(self, img, pad_length):
        """padding_image_overlap (split2process.py:6-13) on the device: h x (w + 2*pad_length) x 3, zero columns each side."""
        h, w = int(img.shape[0]), int(img.shape[1])
        raw = img if img.is_cuda else img.to(self.tdevice, non_blocking=True)
        padded = torch.zeros((h, w + 2 * pad_length, 3), dtype=torch.uint8, device=self.tdevice)
        padded[:, pad_length:pad_length + w] = raw
        return padded

    def crop_frames(self, padded, boxes, frames):
        """frames[i] = img_preprocess(padded[t:b, l:r]) for box i: one b200romp_preprocess_bgr_batch call for all the boxes,
        each crop a window of the padded image (its own size, the padded row stride)."""
        crops = [padded[t:b, l:r] for l, r, t, b in np.asarray(boxes).tolist()]
        preprocess_bgr_batch(self.lib, crops, [None] * len(crops), None, frames, None, self.stream.cuda_stream)

    def crop_post(self, nb, crop0, tab_dev):
        """SMPL-A / SMIL on the chunk's persons, then the per-crop stage (b200romp_bev_crop_post): survivors appended to
        the image-level rows."""
        lib, b, lb, st = self.lib, self.buf, self._long, self.stream.cuda_stream
        cap = nb * MAX_PERSON
        self.smpla.forward(b["betas"], b["thetas"], cap, b["count"], True, b["smpl_ws"], b["verts"], b["joints"], st)
        self.smil.forward(b["betas"], b["thetas"], cap, b["count"], True, b["smpl_ws"], b["verts_smil"], b["joints_smil"], st)
        _lib.check(lib.b200romp_bev_crop_post(
            _ptr(b["betas"]), _ptr(b["verts_smil"]), _ptr(b["joints_smil"]), _ptr(b["verts"]), _ptr(b["joints"]),
            _ptr(b["thetas"]), _ptr(b["params_pred"]), _ptr(b["conf"]), _ptr(b["cam"]), _ptr(b["cam_trans"]),
            _ptr(b["batch_ids"]), nb, cap, _ptr(b["count"]), _ptr(tab_dev), crop0, float(self.settings.relative_scale_thresh),
            _ptr(b["pj2d_org"]), _ptr(b["keep"]), _ptr(b["sel"]), _ptr(lb["cam_full"]), lb["cam"].shape[0], _ptr(lb["count"]),
            _ptr(lb["ctl"]), _ptr(lb["verts"]), _ptr(lb["joints"]), _ptr(lb["thetas"]), _ptr(lb["betas"]),
            _ptr(lb["params_pred"]), _ptr(lb["conf"]), _ptr(lb["cam"]), C.c_void_p(st)), "bev_crop_post")

    @torch.no_grad()
    def long_merge(self, pad_info, img_max_side):
        """Merged stage of the long-image mode (bev/main.py:253-256) on the accumulated rows, then row compaction."""
        lib, lb, sp = self.lib, self._long, C.c_void_p(self.stream.cuda_stream)
        rows = lb["cam"].shape[0]
        off = (C.c_float * 6)(*[float(v) for v in pad_info])
        _lib.check(lib.b200romp_bev_long_merge(_ptr(lb["cam"]), _ptr(lb["joints"]), _ptr(lb["conf"]), rows, _ptr(lb["count"]), off,
                                               float(self.settings.nms_thresh), float(self.settings.relative_scale_thresh),
                                               float(img_max_side), _ptr(lb["cam_trans"]), _ptr(lb["pj2d_org"]), _ptr(lb["removed"]),
                                               _ptr(lb["ws"]), _ptr(lb["sel"]), _ptr(lb["count2"]), sp), "bev_long_merge")
        for k, dst in lb["out"].items():
            src = lb[k]
            row = src[0].numel() * src.element_size()
            _lib.check(lib.b200romp_gather_rows(_ptr(src), row, _ptr(lb["sel"]), _ptr(lb["count2"]), rows, _ptr(dst), sp), "gather_rows")

    def _collect_long(self, to_numpy=True):
        lb = self._long
        n_det, n = self._counts(lb["count"][1:2], lb["count2"])      # persons detected in any crop, persons kept
        if n_det == 0:                        # the reference raises KeyError here (main.py:253); INTEGRATION.md, Deviations
            print("No person detected!")
            return None
        return self._result(lb["out"], n, torch.zeros(n, dtype=torch.int64, device=self.tdevice), to_numpy)

    @torch.no_grad()
    def forward(self, image, signal_ID=0, **kwargs):
        """image: HxWx3 uint8 BGR.  bev/main.py:139-156: crowd mode (the default) takes images with w/h >= 2 through
        ``process_long_image``, every other image through one 512x512 frame."""
        if image.shape[1] / image.shape[0] >= 2 and self.settings.crowd:
            if getattr(self.settings, "show_patch_results", False):
                raise NotImplementedError("show_patch_results renders and saves per-crop images; rendering is out of scope")
            return self.process_long_image(image)
        inp, pad = img_preprocess(image)
        out = self.forward_batch(torch.from_numpy(inp), offsets=pad, img_max_side=float(max(image.shape[:2])), signal_IDs=[signal_ID])
        if out is None:
            print("No person detected!")                                       # bev/model.py:239
            return None
        return out

    def __del__(self):
        try:
            if getattr(self, "h", None):
                self.lib.b200romp_bev_destroy(self.h)
            if getattr(self, "trk", None):
                self.lib.b200romp_bev_tracker_destroy(self.trk)
        except Exception:
            pass
