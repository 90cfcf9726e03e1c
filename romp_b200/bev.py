"""Drop-in call surface of ``simple_romp``'s BEV (bev/main.py) on the GPU hot path.

``bev_settings`` mirrors bev/main.py:27-87 (same flags and defaults, including the quirk that ``crowd`` defaults to
True and therefore overrides the thresholds with ``long_conf_dict``), ``BEV(settings)(image_bgr) -> dict | None``
mirrors bev/main.py:91-258: normal images run as one 512x512 frame, and in crowd mode images at least twice as wide as
high run through ``process_long_image`` (the reference's overlapping crops, batched through the model, with the per-crop
and merged filters on the device; ``process_long_images`` for a list of them, in passes of several images).  ``forward_batch`` is the batched entry point for normal frames, ``forward_images`` the
batched ``forward`` on raw images of different sizes (each frame with its own geometry); ``forward_batches`` and
``forward_image_batches`` stream them on two slots, staging and reading back neighbouring chunks while a chunk's kernels run.
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
from .streams import MAX_VIDEO_STREAMS, StreamFailed, check_streams, check_video_streams, stream_indices
from .staging import RawStager, after_producers, frame_buffer, frame_offsets, image_tensor, preprocess_bgr_batch, to_caller

conf_dict = {1: [0.25, 20, 2], 2: [0.1, 20, 1.6]}                    # bev/main.py:24-25
long_conf_dict = {1: [0.12, 20, 1.5, 0.46], 2: [0.08, 20, 1.6, 0.8]}
model_dict = {1: "BEV_ft_agora.pth", 2: "BEV.pth"}
N_PARAMS = 146                                                       # 3 cam + 22*6 + 11 betas, bev/model.py:116
TRACKER_MAX_TRACKS = 128                                             # live tracks (tracked + lost) of the video mode
MAX_SIGNALS = 4                                                      # filter sets of the video mode, the oldest evicted
LARGEST_KEYS = ("params_pred", "center_confs", "pred_batch_ids")     # --show_largest: one row per detection, not per output


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
    # --- additions of this implementation (the reference has no equivalents)
    p.add_argument("--video_streams", type=int, default=0,
                   help=f"with -t: track up to N independent videos (one per signal_ID, each with its own tracker, ids and "
                        f"filters), stepped in parallel on the GPU; 0 = one tracker shared by every signal_ID, like the "
                        f"reference (at most {MAX_VIDEO_STREAMS})")
    p.add_argument("--inputs", type=str, nargs="+", default=None,
                   help="--mode video on many videos / frame folders in one process (instead of -i): input p writes into "
                        "<save_path>/<stem of p>/ what -i p -o <save_path>/<stem of p> writes; with -t each input is its "
                        "own stream")
    p.add_argument("--open_inputs", type=int, default=8,
                   help="--inputs: how many inputs are read at once (cli.OPEN_INPUTS); the others open in order")
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


def long_images_plan(shapes, overlap_ratio, max_crops):
    """``long_image_plan`` of every (h, w) in ``shapes``, concatenated in list order, and the list cut into passes.

    Returns a dict: boxes int32 [K,4] (every image's boxes in order: the global crop sequence), image int64 [K] (the image
    of each crop), first_crop int64 [n+1] (image j's crops are first_crop[j] .. first_crop[j+1]-1), row_base int64 [n] (64
    x its first crop: where its accumulated rows start), pad_length [n], pad_info fp32 [n,6], img_max_side [n] (max(h, w))
    and passes [(i0, i1)]: images i0 .. i1-1, whole images in list order while their crops total at most
    max(max_crops, K of the pass's first image), so an image with more crops than max_crops is a pass of its own."""
    plans = [long_image_plan(h, w, overlap_ratio) for h, w in shapes]
    counts = [len(p[1]) for p in plans]
    first = np.cumsum([0] + counts)
    passes, i0 = [], 0
    while i0 < len(shapes):
        i1, total = i0 + 1, counts[i0]
        while i1 < len(shapes) and total + counts[i1] <= max(max_crops, counts[i0]):
            total += counts[i1]
            i1 += 1
        passes.append((i0, i1))
        i0 = i1
    return dict(boxes=np.concatenate([p[1] for p in plans]).astype(np.int32) if plans else np.zeros((0, 4), np.int32),
                image=np.repeat(np.arange(len(shapes)), counts), first_crop=first, row_base=MAX_PERSON * first[:-1],
                pad_length=[p[0] for p in plans], pad_info=np.array([p[2] for p in plans], np.float32).reshape(-1, 6),
                img_max_side=[max(h, w) for h, w in shapes], passes=passes)


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
        self.video_streams = check_video_streams(s, self.temporal)
        # NB the reference renders by default (render_mesh is store_false, bev/main.py:44); rendering is out of scope and
        # simply not performed here.
        self.lib = _lib.load()
        self.device_index = int(s.GPU)
        self.tdevice = torch.device("cuda", self.device_index)
        torch.cuda.set_device(self.tdevice)
        self.precision = getattr(s, "precision", "bf16")
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
        # shared scratch: only touched by kernels on self.stream, in order
        self.shared = dict(
            maps_fv=z(B, 4, 128, 128), fv_feats=z(B, 128, 128, 128, dtype=act), img_feats=z(B, 128, 128, graph.bev_feats_channels(self.precision), dtype=act),
            bv_in=z(B, 1, 128, 2560, dtype=act), bv_out=z(B, 1, 128, 128, dtype=act),
            c3d_tmp=z(B, 64, 128, 128), center3d=z(B, 64, 128, 128),
            parse_ws=torch.zeros(int(self.lib.b200romp_bev_parse_workspace_bytes(B)), dtype=torch.uint8, device=dev),
            czyx=z(cap, 3, dtype=i64), cam_czyx=z(cap, 3, dtype=i64), pj2d_org=z(cap, 71, 2), keep=z(cap, dtype=i32), sel=z(cap, dtype=i32))
        if self.calc_smpl:
            self.shared.update(verts=z(cap, 6890, 3), joints=z(cap, 71, 3), verts_smil=z(cap, 6890, 3), joints_smil=z(cap, 71, 3),
                               smpl_ws=z(cap, self.smpla.ws_floats))
        # two slots of what a result reads (the regressor's rows, the compacted rows after the per-frame post filters), with
        # their frames, staging and events, so that chunk i+1 is staged and chunk i-1 read back while chunk i's kernels run
        self.slots = []
        for _ in range(2):
            d = dict(count=z(1, dtype=i32), batch_ids=z(cap, dtype=i64), conf=z(cap), params_pred=z(cap, N_PARAMS), cam=z(cap, 3),
                     thetas=z(cap, 72), betas=z(cap, 11), cam_trans=z(cap, 3), count2=z(1, dtype=i32))
            rows = {**self.shared, **d}
            keys = ("batch_ids", "conf", "params_pred", "cam", "thetas", "betas", "cam_trans", "pj2d_org") + (("verts", "joints") if self.calc_smpl else ())
            # -t reads the tracker's compacted rows (tout): one set of these serves both slots, for direct run_post calls
            out = self.slots[0]["out"] if self.temporal and self.slots else {k: torch.zeros_like(rows[k]) for k in keys}
            self.slots.append(dict(dev=d, out=out, frames={}, pad=z(B, 6), raw=RawStager(dev), done=torch.cuda.Event(),
                                   h2d=torch.cuda.Event(), counts_host=torch.zeros(6 + B, dtype=i32).pin_memory(), host={}))
        self._slot = 0
        self.copy_stream = torch.cuda.Stream(device=dev)
        self.d2h_stream = torch.cuda.Stream(device=dev)

    @property
    def buf(self):
        """device buffers of the slot used by the most recent chunk (+ the shared scratch)"""
        return {**self.shared, **self.slots[self._slot]["dev"]}

    @property
    def out(self):
        """compacted rows (after the per-frame post filters) of the slot used by the most recent chunk"""
        return self.slots[self._slot]["out"]

    @property
    def tbuf(self):
        """-t: the track step's rows of the slot used by the most recent chunk (+ the shared scratch)"""
        return {**self.tshared, **self.slots[self._slot]["tdev"]}

    @property
    def tout(self):
        """-t: the compacted rows of the slot used by the most recent chunk"""
        return self.slots[self._slot]["tout"]

    def _alloc_temporal(self, B):
        """The video mode (bev/main.py:109-121,260-287): one tracker per instance (shared by every signal_ID), the
        filter sets of MAX_SIGNALS signals, and per slot row buffers for up to 2 x 64 rows per frame."""
        dev, R = self.tdevice, 2 * B * MAX_PERSON
        if self.video_streams:                         # stream mode: one tracker per signal_ID
            self.trk = self.lib.b200romp_bev_tracker_create_streams(self.device_index, TRACKER_MAX_TRACKS, self.video_streams)
        else:
            self.trk = self.lib.b200romp_bev_tracker_create(self.device_index, TRACKER_MAX_TRACKS, MAX_SIGNALS)
        if not self.trk:
            raise RuntimeError("b200romp_bev_tracker_create: " + self.lib.b200romp_last_error().decode())
        self.signals = {}                              # signal_ID -> filter set (stream mode: stream index), oldest first
        z = lambda *shape, dtype=torch.float32: torch.zeros(*shape, dtype=dtype, device=dev)
        i64, i32 = torch.int64, torch.int32
        self.tshared = dict(det=z(R, dtype=i32), pj2d_org=z(R, 71, 2), keep=z(R, dtype=i32), sel=z(R, dtype=i32))
        if self.calc_smpl:
            self.tshared.update(verts=z(R, 6890, 3), joints=z(R, 71, 3), verts_smil=z(R, 6890, 3), joints_smil=z(R, 71, 3),
                                smpl_ws=z(R, self.smpla.ws_floats))
        for slot in self.slots:
            # status: the kernel's status, frame_id and rows per frame
            t = dict(count=z(1, dtype=i32), batch_ids=z(R, dtype=i64), track_ids=z(R, dtype=i32), thetas=z(R, 72), betas=z(R, 11),
                     cam=z(R, 3), cam_trans=z(R, 3), params_pred=z(R, N_PARAMS), conf=z(R), status=z(2 + B, dtype=i32),
                     sig=z(B, dtype=i32), count2=z(1, dtype=i32))
            rows = {**self.tshared, **t}
            keys = ("batch_ids", "track_ids", "conf", "params_pred", "cam", "thetas", "betas", "cam_trans", "pj2d_org") + \
                (("verts", "joints") if self.calc_smpl else ())
            slot.update(tdev=t, tout={k: torch.zeros_like(rows[k]) for k in keys}, sig_host=torch.zeros(B, dtype=i32).pin_memory(),
                        sig_h2d=torch.cuda.Event())
        self.frame_id = 0                              # tracker frames so far (frames with a detection)

    def _signal_slots(self, signal_IDs):
        """filter set of every frame's signal_ID; a new signal beyond MAX_SIGNALS evicts the oldest one (its filters are
        reset on the stream, before the batch's kernel).  Stream mode: the stream index of every frame's signal_ID."""
        if self.video_streams:
            return stream_indices(self.signals, signal_IDs, self.video_streams,
                                  lambda k: _lib.check(self.lib.b200romp_bev_tracker_reset(self.trk, k, C.c_void_p(self.stream.cuda_stream)),
                                                       "tracker_reset"))
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

    def _check_streams(self, signal_IDs):
        """Stream mode: raise ValueError, before anything is enqueued, when signal_IDs would make more than
        --video_streams streams live."""
        if self.video_streams:
            check_streams(self.signals, [0] if signal_IDs is None else signal_IDs, self.video_streams)

    def reset_temporal(self, signal_ID=None):
        """Forget every track, id and filter (a new video); ids start again from 1.  Stream mode (--video_streams) with a
        ``signal_ID``: forget that stream only (its index is freed; when the signal_ID comes back its ids start at 1)."""
        if not self.temporal:
            raise RuntimeError("reset_temporal: this BEV instance was built without -t/--temporal_optimize")
        if signal_ID is not None:
            if not self.video_streams:
                raise ValueError("reset_temporal(signal_ID): only in stream mode (--video_streams); the default mode shares "
                                 "one tracker across signal_IDs, reset_temporal() forgets it")
            self.signals.pop(signal_ID, None)          # the index is reset when a signal_ID takes it again
            return
        _lib.check(self.lib.b200romp_bev_tracker_reset(self.trk, -1, C.c_void_p(self.stream.cuda_stream)), "tracker_reset")
        self.signals = {}

    @torch.no_grad()
    def run_temporal(self, B, signal_IDs):
        """BEV.temporal_optimization (bev/main.py:165-169,260-287) of the batch's frames in order: one kernel
        (b200romp_bev_track_step) between the regressor and SMPL-A, writing the smoothed rows to ``self.tbuf``."""
        b, t, slot = self.buf, self.tbuf, self.slots[self._slot]
        slots = self._signal_slots(signal_IDs)
        slot["sids"] = list(signal_IDs)
        slot["sig_h2d"].synchronize()                 # the slot's previous chunk has copied its signal slots
        slot["sig_host"][:B].copy_(torch.tensor(slots, dtype=torch.int32))
        t["sig"][:B].copy_(slot["sig_host"][:B], non_blocking=True)
        slot["sig_h2d"].record(self.stream)
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

    def _result(self, src, n, batch_ids):
        """The output dict (result_keys, plus the SMPL outputs): device views of the first n rows of the buffers ``src``."""
        out = {"smpl_thetas": src["thetas"][:n], "smpl_betas": src["betas"][:n], "cam": src["cam"][:n], "cam_trans": src["cam_trans"][:n],
               "params_pred": src["params_pred"][:n], "center_confs": src["conf"][:n], "pred_batch_ids": batch_ids}
        if self.calc_smpl:
            out.update(verts=src["verts"][:n], joints=src["joints"][:n], pj2d_org=src["pj2d_org"][:n])
        return out

    def _read_back(self, slot, B, to_numpy, temporal, split=False):
        """A chunk's result, on the read-back stream after the slot's kernels: one sync for its row counts (and with
        ``temporal`` the tracker's status), then one more for its valid rows and their frame ids.  Returns None when the
        chunk has no result (nobody detected; with -t no tracker rows), else (out, rows, det, frames): the batch result
        (numpy arrays, views of the slot's pinned mirrors with ``split``, or device views without to_numpy), the frame of
        each of its rows and of each detection (host int64), and the frames that have a result.  Raises on a nonzero
        tracker status."""
        st, d, h = self.d2h_stream, slot["dev"], slot["counts_host"]
        st.wait_event(slot["done"])
        with torch.cuda.stream(st):
            h[0:1].copy_(d["count"], non_blocking=True)
            h[1:2].copy_(d["count2"], non_blocking=True)
            if temporal:
                t = slot["tdev"]
                h[2:3].copy_(t["count"], non_blocking=True)
                h[3:4].copy_(t["count2"], non_blocking=True)
                h[4:6 + B].copy_(t["status"][:2 + B], non_blocking=True)
        st.synchronize()
        n_det, frames = int(h[0]), None
        if temporal:
            n_rows, n_kept, status = int(h[2]), int(h[3]), int(h[4])
            self.frame_id = int(h[5])
            if status and self.video_streams:
                failed = sorted({slot["sids"][b] for b in range(B) if int(h[6 + b]) < 0}, key=repr)
                raise StreamFailed(f"BEV video mode: more than {TRACKER_MAX_TRACKS} live tracks in the stream(s) of signal_ID "
                                   f"{', '.join(map(repr, failed))}; call reset_temporal(signal_ID) for each (the other "
                                   "streams of the batch were tracked)", failed)
            if status:
                raise RuntimeError("BEV video mode: " + (f"more than {TRACKER_MAX_TRACKS} live tracks" if status == 1 else "too many rows")
                                   + "; call reset_temporal() before the next frame")
            frames = [b for b in range(B) if int(h[6 + b])]              # frames the tracker gave rows (before the filters)
            if not frames:
                return None
            src, n = (slot["tout"], n_kept) if self.calc_smpl else (t, n_rows)
        elif n_det == 0:
            return None
        else:
            src, n = (slot["out"], int(h[1])) if self.calc_smpl else (d, n_det)
        out = self._result(src, n, src["batch_ids"][:n])
        if temporal and self.show_largest:           # bev/main.py:262-267: only thetas / betas / cam are cut to one row
            out.update(params_pred=d["params_pred"][:n_det], center_confs=d["conf"][:n_det], pred_batch_ids=d["batch_ids"][:n_det])
        elif temporal:
            out["track_ids"] = src["track_ids"][:n]
        ids = dict(_rows=src["batch_ids"][:n], _det=d["batch_ids"][:n_det])
        # a result split per frame is copied out of pinned mirrors frame by frame; a whole-batch result goes straight
        # into arrays of its own (a mirror would cost it a second host copy)
        fetch = {**ids, **out} if to_numpy and split else ids
        host = slot["host"]
        with torch.cuda.stream(st):
            for k, v in fetch.items():
                if k not in host or len(host[k]) < len(v):      # pinned mirrors, allocated on first use, grown on demand
                    rows = max(len(v), 2 * len(host.get(k, ())), 64)
                    host[k] = torch.empty((rows, *v.shape[1:]), dtype=v.dtype, pin_memory=True)
                host[k][:len(v)].copy_(v, non_blocking=True)
            if to_numpy and not split:
                out = {k: v.cpu().numpy() for k, v in out.items()}
        st.synchronize()
        got = {k: host[k][:len(v)].numpy() for k, v in fetch.items()}
        if to_numpy and split:
            out = {k: got[k] for k in out}
        if frames is None:
            frames = np.unique(got["_det"]).tolist()
        return out, got["_rows"], got["_det"], frames

    @staticmethod
    def _batch(got):
        """forward_batch's dict from a read-back: host arrays, or device views"""
        return None if got is None else got[0]

    def _per_frame(self, got, B, to_numpy, slot):
        """forward_images' per-frame dicts from a chunk's read-back in ``slot``: None for a frame without a result, else
        the frame's rows of every key (arrays that own their memory, or device copies on the caller's stream) with
        pred_batch_ids zeroed.  The rows come in frame order, so each frame's rows are one host searchsorted on their
        frame ids."""
        res = [None] * B
        if got is None:
            return res
        out, rows, det, frames = got
        br = np.searchsorted(rows, np.arange(B + 1)).tolist()
        bd = np.searchsorted(det, np.arange(B + 1)).tolist()
        largest = LARGEST_KEYS if self.temporal and self.show_largest else ()
        for f in frames:
            r = {}
            for k, v in out.items():
                s, e = (bd[f], bd[f + 1]) if k in largest else (br[f], br[f + 1])
                r[k] = np.array(v[s:e]) if to_numpy else v[s:e]
            res[f] = r
        if not to_numpy:
            res = to_caller(res, slot["done"], self.stream)
        for r in res:
            if r is not None:
                if to_numpy:
                    r["pred_batch_ids"] = np.zeros(len(r["pred_batch_ids"]), np.int64)
                else:
                    r["pred_batch_ids"].zero_()
        return res

    def collect(self, to_numpy=True):
        """The result of the frames that run_model / run_post last enqueued on self.stream (the current slot, without the
        video mode's tracker rows): one dict with pred_batch_ids, or None when nobody was detected."""
        slot = self.slots[self._slot]
        slot["done"].record(self.stream)
        return self._batch(self._read_back(slot, 0, to_numpy, False))

    def _next_slot(self):
        self._slot ^= 1
        return self.slots[self._slot]

    def _run(self, slot, fd, B, offsets, img_max_side, center3d_override, signal_IDs):
        """A chunk's kernels on self.stream after its frames fd: model, with -t the track step, post filters; then the
        slot's done event (also when a chunk is refused on the way: the slot is free after what was enqueued)."""
        try:
            self.run_model(fd, center3d_override)
            if self.temporal:
                self.run_temporal(B, [0] * B if signal_IDs is None else list(signal_IDs))
                self.run_post_temporal(B, offsets, img_max_side)
            else:
                self.run_post(B, offsets, img_max_side)
        finally:
            slot["done"].record(self.stream)

    @torch.no_grad()
    def forward_batch(self, frames, offsets=None, to_numpy=True, center3d_override=None, img_max_side=512.0, signal_IDs=None):
        """frames [B,512,512,3] padded+resized like img_preprocess.  ``offsets``: one pad info [top,bottom,left,right,h,w]
        for every frame, suppressing with ``img_max_side``; or one row per frame ([B,6], numpy or tensor), each frame then
        suppressing with its own max(h, w) (``img_max_side`` is not used).  With -t the frames are consecutive video
        frames, tracked and smoothed in order (``signal_IDs``: one per frame, default 0); the result adds ``track_ids``.
        With --video_streams every signal_ID is an independent video (its own tracker, ids from 1 and filters,
        romp_b200/streams.py), stepped in parallel; this holds for every video entry point.
        ``to_numpy=False`` returns device tensors of the caller's current stream (see forward_batches)."""
        sids = None if signal_IDs is None else [signal_IDs]
        return next(self.forward_batches([frames], offsets, center3d_override, to_numpy, img_max_side, sids))

    @torch.no_grad()
    def forward_batches(self, batches, offsets=None, center3d_override=None, to_numpy=True, img_max_side=512.0, signal_IDs=None):
        """Streaming form of ``forward_batch`` over an iterable of frame batches [B,512,512,3] (a video): yields what
        ``forward_batch`` returns for each batch, in order.  Each batch goes into the next of two slots: its frames are
        copied into the slot's frame buffer on the copy stream, so the copy of batch i+1 and the read-back of batch i-1
        overlap the kernels of batch i.  The generator goes on once a host batch has been copied, so a caller may refill
        one (pinned or numpy) buffer in place between batches.  ``offsets``, ``center3d_override`` and ``img_max_side``
        apply to every batch; with -t the batches are consecutive parts of one video and ``signal_IDs`` is None or one
        sequence per batch.  Device-resident frames, ``center3d_override`` and per-frame ``offsets`` may come from
        producers on the caller's current stream (the model's streams wait for it) and may be dropped once handed over.
        The yielded results own their memory: arrays, or with ``to_numpy=False`` copies made on the caller's current
        stream after the batch's kernels, which the caller may read there at any later time (the model's kernels wait
        for the copies before they reuse the slot)."""
        after_producers(self.stream, self.tdevice, center3d_override, offsets)
        sid_iter = None if signal_IDs is None else iter(signal_IDs)
        pending = None
        for frames in batches:
            slot = self._submit_frames(frames, offsets, center3d_override, img_max_side, None if sid_iter is None else next(sid_iter))
            if pending is not None:
                yield self._batch_result(*pending, to_numpy)
            pending = slot
        if pending is not None:
            yield self._batch_result(*pending, to_numpy)

    def _batch_result(self, slot, B, to_numpy):
        """A batch's result for the caller: arrays (to_numpy), else copies of the slot's rows on the caller's stream."""
        out = self._batch(self._read_back(slot, B, to_numpy, self.temporal))
        return out if out is None or to_numpy else to_caller([out], slot["done"], self.stream)[0]

    def _submit_frames(self, frames, offsets, center3d_override, img_max_side, signal_IDs):
        """One batch of frames into the next slot; returns (slot, B) once host frames have been copied."""
        if isinstance(frames, np.ndarray):
            frames = torch.from_numpy(frames)
        B = frames.shape[0]
        self._check_streams(signal_IDs)
        slot = self._next_slot()
        fd = frame_buffer(slot["frames"], frames.dtype, B, self.tdevice)
        after_producers(self.copy_stream, self.tdevice, frames)
        with torch.cuda.stream(self.copy_stream):
            self.copy_stream.wait_event(slot["done"])          # the slot's previous kernels no longer read fd
            fd.copy_(frames, non_blocking=True)
            slot["h2d"].record(self.copy_stream)
        with torch.cuda.stream(self.stream):
            self.stream.wait_event(slot["h2d"])
            self._run(slot, fd, B, frame_offsets(offsets, slot["pad"], B), img_max_side, center3d_override, signal_IDs)
        if not frames.is_cuda:
            slot["h2d"].synchronize()
        return slot, B

    @torch.no_grad()
    def forward_images(self, images, to_numpy=True, center3d_override=None, signal_IDs=None):
        """Batched ``forward`` on raw images of any sizes (HxWx3 uint8 BGR: numpy arrays, host or device tensors): a list
        of the same length, element i the result for images[i] (dict or None; nothing is printed for normal images).
        Normal images run in chunks of at most ``max_batch`` through one preprocessing kernel per chunk (the GPU kernel,
        not the host OpenCV resize of ``forward``) and b200romp_bev_post_frames, each frame with its own pad info and
        suppression threshold; element i then equals ``forward_batch`` on image i's GPU-preprocessed frame with its pad
        info and ``img_max_side = max(h, w)``.  A frame with a detection whose persons were all filtered out gives a dict
        of empty arrays.  In crowd mode the images with w/h >= 2 go together through ``process_long_images``.
        center3d_override: optional device [n_normal,64,128,128] for the normal images in order.
        With -t the normal images are consecutive video frames (``signal_IDs``: one per image, default 0), tracked and
        smoothed in list order; wide crowd-mode images are neither tracked nor smoothed (bev/main.py:140-143)."""
        sids = None if signal_IDs is None else [signal_IDs]
        return next(self.forward_image_batches([images], to_numpy, center3d_override, sids))

    @torch.no_grad()
    def forward_image_batches(self, batches, to_numpy=True, center3d_override=None, signal_IDs=None):
        """Streaming form of ``forward_images`` over an iterable of image lists: yields, for each list, what
        ``forward_images`` returns for it, in order.  Each chunk of at most ``max_batch`` normal images is staged into
        its slot's pinned buffer and sent with one H2D on the copy stream (device images are read in place), so staging
        chunk i+1 and reading back chunk i-1 overlap the kernels of chunk i (the two slots of ``forward_batches``).  A
        list's wide crowd-mode images drain the pipeline once and run through one ``process_long_images`` call (one host
        sync per pass) before the list's first chunk.
        center3d_override applies to every list, entry k to the k-th normal image of the list.  With -t the lists are
        consecutive parts of one video (tracker and filters carry across them) and ``signal_IDs`` is None or one sequence
        per list.  Host images have been staged when the generator pulls the next list; device images and
        ``center3d_override`` may come from producers on the caller's current stream.  The yielded results own their
        memory, as in ``forward_batches``."""
        if center3d_override is not None:
            assert center3d_override.is_cuda
        after_producers(self.stream, self.tdevice, center3d_override)
        sid_iter = None if signal_IDs is None else iter(signal_IDs)

        def chunks():
            """(images, signal IDs, result list, the chunk's normal images, their 3-D centre maps, the wide images to run
            before the chunk (all of the list's, before its first chunk), last chunk of the list)"""
            for images in batches:
                imgs = [image_tensor(x) for x in images]
                sids = [0] * len(imgs) if sid_iter is None else list(next(sid_iter))
                if len(sids) != len(imgs):
                    raise ValueError(f"forward_image_batches: {len(sids)} signal_IDs for {len(imgs)} images")
                wide = [i for i, t in enumerate(imgs) if self.settings.crowd and t.shape[1] / t.shape[0] >= 2]
                normal = [i for i in range(len(imgs)) if i not in set(wide)]
                if self.temporal:
                    self._check_streams([sids[i] for i in normal])
                if wide and getattr(self.settings, "show_patch_results", False):
                    raise NotImplementedError("show_patch_results renders and saves per-crop images; rendering is out of scope")
                if center3d_override is not None:
                    assert center3d_override.shape[0] >= len(normal)
                res = [None] * len(imgs)
                for c0 in range(0, max(len(normal), 1), self.max_batch):
                    idx = normal[c0:c0 + self.max_batch]
                    last = c0 + self.max_batch >= len(normal)
                    co = None if center3d_override is None or not idx else center3d_override[c0:c0 + len(idx)]
                    yield imgs, sids, res, idx, co, wide if c0 == 0 else [], last

        pending = None
        for imgs, sids, res, idx, co, wide, last in chunks():
            if wide and pending is not None:       # drain: the long-image mode runs in the current slot's rows
                done = self._finish_images(*pending, to_numpy)
                pending = None
                if done is not None:
                    yield done
            if wide:
                for i, r in zip(wide, self.process_long_images([imgs[i] for i in wide], to_numpy=to_numpy)):
                    res[i] = r
            slot = self._submit_images([imgs[i] for i in idx], co, [sids[i] for i in idx]) if idx else None
            if pending is not None:
                done = self._finish_images(*pending, to_numpy)
                if done is not None:
                    yield done
            pending = (slot, res, idx, last)
        if pending is not None:
            yield self._finish_images(*pending, to_numpy)

    def _submit_images(self, imgs, center3d_override, signal_IDs):
        """One chunk of normal images into the next slot: host images staged into its pinned buffer and sent with one H2D
        on the copy stream, one preprocessing kernel into its frames and pad table, then the chunk's kernels."""
        B = len(imgs)
        slot = self._next_slot()
        fd = frame_buffer(slot["frames"], torch.uint8, B, self.tdevice)
        raw = slot["raw"]
        offs, total = raw.stage(imgs, replace_after=slot["done"], reuse_after=slot["h2d"])
        if total:
            with torch.cuda.stream(self.copy_stream):
                self.copy_stream.wait_event(slot["done"])      # the slot's previous preprocessing no longer reads raw.dev
                raw.upload(total)
                slot["h2d"].record(self.copy_stream)
            self.stream.wait_event(slot["h2d"])
        after_producers(self.stream, self.tdevice, *imgs)
        with torch.cuda.stream(self.stream):
            preprocess_bgr_batch(self.lib, imgs, offs, raw.dev, fd, slot["pad"], self.stream.cuda_stream)
            self._run(slot, fd, B, slot["pad"][:B], 512.0, center3d_override, signal_IDs)
        return slot

    def _finish_images(self, slot, res, idx, last, to_numpy):
        """Read back one chunk into res at its images' places; returns res once its list's last chunk is in."""
        if slot is not None:
            for i, r in zip(idx, self._per_frame(self._read_back(slot, len(idx), to_numpy, self.temporal, True), len(idx), to_numpy, slot)):
                res[i] = r
        return res if last else None

    def _long_buffers(self, rows, n_images=1):
        """Accumulation rows of the long-image mode for a pass of up to n_images images (grown on demand, kept for the
        next pass)."""
        lb = getattr(self, "_long", None)
        if lb is not None and lb["cam"].shape[0] >= rows and lb["img_sel"].shape[0] >= n_images:
            return lb
        if lb is not None:
            rows, n_images = max(rows, lb["cam"].shape[0]), max(n_images, lb["img_sel"].shape[0])
        dev = self.tdevice
        z = lambda *shape, dtype=torch.float32: torch.zeros(*shape, dtype=dtype, device=dev)
        lb = dict(verts=z(rows, 6890, 3), joints=z(rows, 71, 3), thetas=z(rows, 72), betas=z(rows, 11), params_pred=z(rows, N_PARAMS),
                  conf=z(rows), cam=z(rows, 3), cam_trans=z(rows, 3), pj2d_org=z(rows, 71, 2), removed=z(rows, dtype=torch.int32),
                  sel=z(rows, dtype=torch.int32), count=z(2 * n_images, dtype=torch.int32), count2=z(1, dtype=torch.int32),
                  img_sel=z(n_images, 2, dtype=torch.int32), ctl=z(2 * self.max_batch, dtype=torch.int32), cam_full=z(self.cap, 3),
                  ws=torch.zeros(int(self.lib.b200romp_bev_long_merge_images_workspace_bytes(rows, n_images)), dtype=torch.uint8,
                                 device=dev),
                  host=torch.zeros(4 * n_images, dtype=torch.int32).pin_memory(), done=torch.cuda.Event())
        lb["out"] = {k: torch.zeros_like(lb[k]) for k in ("verts", "joints", "thetas", "betas", "params_pred", "conf", "cam",
                                                          "cam_trans", "pj2d_org")}
        self._long = lb
        return lb

    @torch.no_grad()
    def process_long_image(self, full_image, center3d_override=None, to_numpy=True):
        """Crowd mode for one image at least twice as wide as high, bev/main.py:184-258 (``BEV.forward`` dispatches
        here): ``process_long_images([full_image])[0]``.  center3d_override: optional device [K,64,128,128] replacing
        the crops' 3-D centre maps (tests, measurement)."""
        return self.process_long_images([full_image], center3d_override, to_numpy)[0]

    @torch.no_grad()
    def process_long_images(self, images, center3d_override=None, to_numpy=True):
        """Crowd mode for a list of images, each at least twice as wide as high (HxWx3 uint8 BGR: numpy arrays, host or
        device tensors): element i is ``process_long_image(images[i])`` bit for bit, a dict, or None after printing
        "No person detected!".

        Every image is zero-padded horizontally on the device and cut into the reference's overlapping crops
        (``long_images_plan``).  The list runs in passes of whole images (at most max(2 x max_batch, K of the pass's first
        image) crops): a pass's crops, image after image, become 512x512 frames (b200romp_preprocess_bgr_batch on the
        crops' windows of the padded images) and run through the model in chunks of at most ``max_batch`` frames that
        may hold crops of several images; each chunk's persons go through the per-crop filters and are appended to their
        own image's rows (b200romp_bev_crop_post_images), and the merged filters run on every image of the pass at once
        (b200romp_bev_long_merge_images).  One host sync per pass.  center3d_override: optional device [sum K,64,128,128]
        replacing the crops' 3-D centre maps, in crop order, image by image (tests, measurement).  ``to_numpy=False``
        returns device tensors of the caller's current stream that own their memory (see forward_batches)."""
        if not self.calc_smpl:
            raise ValueError("the long-image mode needs SMPL (bev/main.py:203): calc_smpl must be on for images with w/h >= 2")
        imgs = [image_tensor(x) for x in images]
        if not imgs:
            return []
        shapes = [(int(t.shape[0]), int(t.shape[1])) for t in imgs]
        if any(w / h < 2 for h, w in shapes):
            raise ValueError(f"process_long_images: every image needs w/h >= 2, got (h, w) {shapes}")
        plan = long_images_plan(shapes, self.settings.overlap_ratio, 2 * self.max_batch)
        if center3d_override is not None:
            assert center3d_override.is_cuda and tuple(center3d_override.shape) == (len(plan["boxes"]), 64, 128, 128)
        after_producers(self.stream, self.tdevice, center3d_override, *imgs)
        fc = plan["first_crop"]
        self._long_buffers(max([MAX_PERSON * int(fc[i1] - fc[i0]) for i0, i1 in plan["passes"]], default=0),
                           max([i1 - i0 for i0, i1 in plan["passes"]], default=1))
        res = []
        for i0, i1 in plan["passes"]:
            res += self._long_pass(imgs, plan, i0, i1, center3d_override, to_numpy)
        return res

    def _long_pass(self, imgs, plan, i0, i1, center3d_override, to_numpy):
        """One pass of process_long_images: images i0 .. i1-1 of the plan, their results in order."""
        s, B, dev, lb = self.settings, self.max_batch, self.tdevice, self._long
        fc = plan["first_crop"]
        k0, K, n = int(fc[i0]), int(fc[i1] - fc[i0]), i1 - i0
        boxes, pads = plan["boxes"][k0:k0 + K], plan["pad_length"]
        tab = np.concatenate([long_image_crop_table(plan["boxes"][fc[j]:fc[j + 1]], pads[j], *imgs[j].shape[:2], float(s.nms_thresh))
                              for j in range(i0, i1)])
        base =(plan["row_base"][i0:i1] - plan["row_base"][i0]).astype(np.int32)
        crops = np.stack([plan["image"][k0:k0 + K] - i0, base[plan["image"][k0:k0 + K] - i0]], 1).astype(np.int32)
        host = [torch.from_numpy(a).pin_memory() for a in (tab, crops, plan["pad_info"][i0:i1], base)]
        frames = frame_buffer(self.slots[self._slot]["frames"], torch.uint8, B, dev)           # free: callers drain first
        with torch.cuda.stream(self.stream):
            padded = [self.pad_long_image(imgs[j], pads[j]) for j in range(i0, i1)]
            tab_dev, crops_dev, pad_dev, base_dev = [t.to(dev, non_blocking=True) for t in host]
            lb["count"][:2 * n].zero_()
            for c0 in range(0, K, B):
                nb = min(B, K - c0)
                self.crop_frames([padded[i] for i in crops[c0:c0 + nb, 0]], boxes[c0:c0 + nb], frames)   # main.py:197-199
                self.run_model(frames[:nb], None if center3d_override is None else center3d_override[k0 + c0:k0 + c0 + nb])
                self.crop_post(nb, c0, tab_dev, crops_dev)
            self.long_merge_images(pad_dev, base_dev, MAX_PERSON * int(np.max(np.diff(fc[i0:i1 + 1]))))
        return self._collect_long_images(n, to_numpy)

    def pad_long_image(self, img, pad_length):
        """padding_image_overlap (split2process.py:6-13) on the device: h x (w + 2*pad_length) x 3, zero columns each side."""
        h, w = int(img.shape[0]), int(img.shape[1])
        raw = img if img.is_cuda else img.to(self.tdevice, non_blocking=True)
        padded = torch.zeros((h, w + 2 * pad_length, 3), dtype=torch.uint8, device=self.tdevice)
        padded[:, pad_length:pad_length + w] = raw
        return padded

    def crop_frames(self, padded, boxes, frames):
        """frames[i] = img_preprocess(padded[t:b, l:r]) for box i: one b200romp_preprocess_bgr_batch call for all the boxes,
        each crop a window of the padded image (its own size, the padded row stride).  ``padded``: one padded image, or
        a list with the padded image of every box."""
        padded = padded if isinstance(padded, list) else [padded] * len(boxes)
        crops = [p[t:b, l:r] for p, (l, r, t, b) in zip(padded, np.asarray(boxes).tolist())]
        preprocess_bgr_batch(self.lib, crops, [None] * len(crops), None, frames, None, self.stream.cuda_stream)

    def crop_post(self, nb, crop0, tab_dev, crops_dev=None):
        """SMPL-A / SMIL on the chunk's persons, then the per-crop stage: survivors appended to the image-level rows.
        ``crops_dev``: the pass's device int32 [K,2] {image, first row} table (b200romp_bev_crop_post_images); None for
        the crops of one image (b200romp_bev_crop_post)."""
        lib, b, lb, st = self.lib, self.buf, self._long, self.stream.cuda_stream
        cap = nb * MAX_PERSON
        self.smpla.forward(b["betas"], b["thetas"], cap, b["count"], True, b["smpl_ws"], b["verts"], b["joints"], st)
        self.smil.forward(b["betas"], b["thetas"], cap, b["count"], True, b["smpl_ws"], b["verts_smil"], b["joints_smil"], st)
        rows = (_ptr(b["betas"]), _ptr(b["verts_smil"]), _ptr(b["joints_smil"]), _ptr(b["verts"]), _ptr(b["joints"]),
                _ptr(b["thetas"]), _ptr(b["params_pred"]), _ptr(b["conf"]), _ptr(b["cam"]), _ptr(b["cam_trans"]),
                _ptr(b["batch_ids"]), nb, cap, _ptr(b["count"]), _ptr(tab_dev))
        acc = (crop0, float(self.settings.relative_scale_thresh), _ptr(b["pj2d_org"]), _ptr(b["keep"]), _ptr(b["sel"]),
               _ptr(lb["cam_full"]), lb["cam"].shape[0], _ptr(lb["count"]), _ptr(lb["ctl"]), _ptr(lb["verts"]), _ptr(lb["joints"]),
               _ptr(lb["thetas"]), _ptr(lb["betas"]), _ptr(lb["params_pred"]), _ptr(lb["conf"]), _ptr(lb["cam"]), C.c_void_p(st))
        if crops_dev is None:
            _lib.check(lib.b200romp_bev_crop_post(*rows, *acc), "bev_crop_post")
        else:
            _lib.check(lib.b200romp_bev_crop_post_images(*rows, _ptr(crops_dev), *acc), "bev_crop_post_images")

    @torch.no_grad()
    def long_merge(self, pad_info, img_max_side):
        """Merged stage of the long-image mode (bev/main.py:253-256) on one image's accumulated rows, then row
        compaction: the one-image case of ``long_merge_images`` (b200romp_bev_long_merge, the count kept to img_sel[0])."""
        lb = self._long
        off = (C.c_float * 6)(*[float(v) for v in pad_info])
        _lib.check(self.lib.b200romp_bev_long_merge(
            _ptr(lb["cam"]), _ptr(lb["joints"]), _ptr(lb["conf"]), lb["cam"].shape[0], _ptr(lb["count"]), off,
            float(self.settings.nms_thresh), float(self.settings.relative_scale_thresh), float(img_max_side), _ptr(lb["cam_trans"]),
            _ptr(lb["pj2d_org"]), _ptr(lb["removed"]), _ptr(lb["ws"]), _ptr(lb["sel"]), _ptr(lb["img_sel"][0, 1:]),
            C.c_void_p(self.stream.cuda_stream)), "bev_long_merge")
        self._gather_long(lb["img_sel"][0, 1:])

    @torch.no_grad()
    def long_merge_images(self, pad_dev, base_dev, image_rows):
        """Merged stage of a pass (b200romp_bev_long_merge_images) on the accumulated rows of its images (device pad
        table [n,6], device int32 first rows [n], at most image_rows rows per image), then one row compaction for all."""
        lb = self._long
        _lib.check(self.lib.b200romp_bev_long_merge_images(
            _ptr(lb["cam"]), _ptr(lb["joints"]), _ptr(lb["conf"]), lb["cam"].shape[0], len(base_dev), image_rows, _ptr(base_dev),
            _ptr(lb["count"]), _ptr(pad_dev), float(self.settings.nms_thresh), float(self.settings.relative_scale_thresh),
            _ptr(lb["cam_trans"]), _ptr(lb["pj2d_org"]), _ptr(lb["removed"]), _ptr(lb["ws"]), _ptr(lb["sel"]), _ptr(lb["img_sel"]),
            _ptr(lb["count2"]), C.c_void_p(self.stream.cuda_stream)), "bev_long_merge_images")
        self._gather_long(lb["count2"])

    def _gather_long(self, count):
        """lb["out"][k][i] = lb[k][sel[i]] for i < count (device int32 [1]), one launch per field."""
        lb, sp = self._long, C.c_void_p(self.stream.cuda_stream)
        for k, dst in lb["out"].items():
            src = lb[k]
            row = src[0].numel() * src.element_size()
            _lib.check(self.lib.b200romp_gather_rows(_ptr(src), row, _ptr(lb["sel"]), _ptr(count), src.shape[0], _ptr(dst), sp),
                       "gather_rows")

    def _collect_long(self, to_numpy=True):
        """The result of one image's merged stage (``long_merge``)."""
        return self._collect_long_images(1, to_numpy)[0]

    def _collect_long_images(self, n, to_numpy=True):
        """The results of a pass's n images from its merged stage: one host sync for the persons detected in each image's
        crops and the start and count of its kept rows, then each image's rows (arrays, or copies on the caller's stream)."""
        lb, h = self._long, self._long["host"]
        with torch.cuda.stream(self.stream):
            h[:2 * n].copy_(lb["count"][:2 * n], non_blocking=True)
            h[2 * n:4 * n].copy_(lb["img_sel"][:n].reshape(-1), non_blocking=True)
            lb["done"].record(self.stream)
        self.stream.synchronize()
        det, start, kept = h[1:2 * n:2].tolist(), h[2 * n:4 * n:2].tolist(), h[2 * n + 1:4 * n:2].tolist()
        src = lb["out"]
        if to_numpy:
            with torch.cuda.stream(self.stream):
                src = {k: v[:start[-1] + kept[-1]].cpu().numpy() for k, v in src.items()}
        res = []
        for j in range(n):
            if det[j] == 0:                   # the reference raises KeyError here (main.py:253); INTEGRATION.md, Deviations
                print("No person detected!")
                res.append(None)
                continue
            s, k = start[j], kept[j]
            ids = np.zeros(k, np.int64) if to_numpy else torch.zeros(k, dtype=torch.int64, device=self.tdevice)
            res.append(self._result({key: v[s:] for key, v in src.items()}, k, ids))
        return res if to_numpy else to_caller(res, lb["done"], self.stream)

    @torch.no_grad()
    def forward(self, image, signal_ID=0, **kwargs):
        """image: HxWx3 uint8 BGR.  bev/main.py:139-156: crowd mode (the default) takes images with w/h >= 2 through
        ``process_long_image``, every other image through one 512x512 frame."""
        if image.shape[1] / image.shape[0] >= 2 and self.settings.crowd:
            if getattr(self.settings, "show_patch_results", False):
                raise NotImplementedError("show_patch_results renders and saves per-crop images; rendering is out of scope")
            return self.process_long_image(image)
        inp, pad = img_preprocess(image)
        # the reference suppresses with max(image.shape), channels included (bev/main.py:179)
        out = self.forward_batch(torch.from_numpy(inp), offsets=pad, img_max_side=float(max(*image.shape[:2], 3)), signal_IDs=[signal_ID])
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


DEFAULT_MODEL_ID = 2     # bev/main.py:23; its video-mode prefix names this default, not --model_id (:304)


def check_cli(args):
    """What the ``bev`` command line refuses, before a model is built: display (with the message of ``BEV``) and any
    mode but image and video (webcam capture is not provided).  The default --render_mesh is ignored: nothing renders,
    and the saved PNG is the input frame."""
    if getattr(args, "show", False):
        raise NotImplementedError("display (--show) is outside the GPU hot path (SURVEY.md section 2)")
    if args.mode not in ("image", "video"):
        raise NotImplementedError("webcam capture is outside the hot path; call BEV.forward per frame")
    from .cli import check_inputs
    check_inputs(args)


def main(input_args=None):
    """The ``bev`` command (bev/main.py:289-307) on the batched image path (romp_b200/cli.py).  ``--mode image`` saves
    ``ResultSaver('image', save_path)``'s files with the prefix ``{center_thresh}``; ``--mode video`` saves every frame
    with the prefix ``_{2}_{center_thresh}``, then ``video_results.npz`` and with ``--save_video`` the mp4, for ``-i``
    or for each of ``--inputs``."""
    from . import cli
    args = bev_settings(sys.argv[1:] if input_args is None else input_args)
    check_cli(args)
    bev = BEV(args)
    if args.mode == "video":
        prefix = f"_{DEFAULT_MODEL_ID}_{args.center_thresh}"
        if args.inputs is not None:
            cli.run_inputs_command(bev, args, prefix)
        else:
            cli.run_video(bev, args, prefix=prefix)
        return
    run_image(bev, args.input, args.save_path, args.center_thresh)


def run_image(bev, input_path, save_path, center_thresh, center3d_override=None):
    """``--mode image``: one image through ``run_frames``, saved by ``ResultSaver('image', save_path)`` with the prefix
    ``{center_thresh}`` (bev/main.py:291-296)."""
    from . import cli
    import cv2
    saver = cli.ResultSaver("image", save_path)
    cli.run_frames(bev, [(input_path, cv2.imread(input_path))], saver, f"{center_thresh}", center3d_override)
    return saver


if __name__ == "__main__":
    main()
