"""Drop-in call surface of ``simple_romp``'s ROMP for the per-frame inference hot path.

Mirrors simple_romp/romp/main.py: ``romp_settings`` (:17-60, same flags and defaults, minus the
import-time download side effects), ``class ROMP`` (:64-176) with ``ROMP(settings)(image_bgr) -> dict | None``
and the same output dict (SURVEY section 8b).  ``forward_batch`` is the batched entry point the reference
lacks (its ``forward`` takes one image per call, main.py:106-107).

Python/PyTorch here only allocates device buffers, owns the CUDA stream and moves bytes; every per-frame
FLOP runs in libb200romp.so (hand-written sm_90a CUDA).  There is no CPU or PyTorch compute fallback:
without the library or without a GPU, constructing ``ROMP`` raises.
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
from .streams import MAX_VIDEO_STREAMS, check_video_streams, stream_indices
from .staging import (FULL_FRAME, RawStager, after_producers, frame_buffer, frame_offsets, image_tensor, preprocess_bgr_batch,
                      split_by_frame, to_caller)

MAX_PERSON = 64          # CenterMap.max_person, post_parser.py:11
N_PARAMS = 145           # 3 cam + 22*6 rot6d + 10 betas, model.py:429


def romp_settings(input_args=sys.argv[1:]):
    """Same flags/defaults as the reference's romp_settings (main.py:17-60); no downloads, no prints."""
    parser = argparse.ArgumentParser(description="ROMP (GPU-native hot path)")
    parser.add_argument("-m", "--mode", type=str, default="image")
    parser.add_argument("-i", "--input", type=str, default=None)
    parser.add_argument("-o", "--save_path", type=str, default=osp.join(osp.expanduser("~"), "ROMP_results"))
    parser.add_argument("--GPU", type=int, default=0)
    parser.add_argument("--onnx", action="store_true")
    parser.add_argument("-t", "--temporal_optimize", action="store_true")
    parser.add_argument("--center_thresh", type=float, default=0.25)
    parser.add_argument("--show_largest", action="store_true")
    parser.add_argument("-sc", "--smooth_coeff", type=float, default=3.0)
    parser.add_argument("--calc_smpl", action="store_false")
    parser.add_argument("--render_mesh", action="store_true")
    parser.add_argument("--renderer", type=str, default="sim3dr")
    parser.add_argument("--show", action="store_true")
    parser.add_argument("--show_items", type=str, default="mesh")
    parser.add_argument("--save_video", action="store_true")
    parser.add_argument("--frame_rate", type=int, default=24)
    parser.add_argument("--smpl_path", type=str, default=osp.join(osp.expanduser("~"), ".romp", "SMPL_NEUTRAL.pth"))
    parser.add_argument("--model_path", type=str, default=osp.join(osp.expanduser("~"), ".romp", "ROMP.pkl"))
    parser.add_argument("--model_onnx_path", type=str, default=osp.join(osp.expanduser("~"), ".romp", "ROMP.onnx"))
    parser.add_argument("--root_align", type=bool, default=False)
    parser.add_argument("--webcam_id", type=int, default=0)
    # --- additions of this implementation (the reference has no equivalents)
    parser.add_argument("--precision", type=str, default="bf16", choices=["bf16", "tf32", "fp32"],
                        help="conv arithmetic: bf16 tensor cores (fast), tf32 tensor cores on fp32 tensors (the reference's "
                             "default GPU arithmetic, cudnn.allow_tf32) or fp32 CUDA cores (strict parity)")
    parser.add_argument("--max_batch", type=int, default=64, help="largest batch forward_batch will be given")
    parser.add_argument("--backbone", type=str, default="hrnet32", choices=["hrnet32", "resnet50"],
                        help="hrnet32 = simple_romp's ROMPv1 (model.py); resnet50 = the training package's ResNet-50 variant "
                             "(romp/lib/models/resnet_50.py; workload cfg1), state dict with the same head keys")
    parser.add_argument("--cam_trans", type=str, default="lsq", choices=["lsq", "pnp", "epnp"],
                        help="cam_trans estimator: lsq = closed-form least squares on the GPU (the reference's fallback, "
                             "utils.py:347-389); pnp = the reference's default cv2.solvePnPRansac per person on the host; "
                             "epnp = the reference's RANSAC loop and validity mask on the GPU, with the published EPnP as "
                             "its solver (every entry point)")
    parser.add_argument("--video_streams", type=int, default=0,
                        help=f"with -t: track up to N independent videos (one per signal_ID, each with its own tracker, ids "
                             f"and filters), stepped in parallel on the GPU by forward_video(_batches) and forward; 0 = the "
                             f"per-instance signal table (at most {MAX_VIDEO_STREAMS})")
    parser.add_argument("--inputs", type=str, nargs="+", default=None,
                        help="--mode video on many videos / frame folders in one process (instead of -i): input p writes "
                             "into <save_path>/<stem of p>/ what -i p -o <save_path>/<stem of p> writes; with -t each "
                             "input is its own stream")
    parser.add_argument("--open_inputs", type=int, default=8,
                        help="--inputs: how many inputs are read at once (cli.OPEN_INPUTS); the others open in order")
    args = parser.parse_args(input_args)
    if not os.path.exists(args.smpl_path):
        alt = args.smpl_path.replace("SMPL_NEUTRAL.pth", "smpl_packed_info.pth")   # main.py:50-52
        if os.path.exists(alt):
            args.smpl_path = alt
    return args


def padding_image(image):
    """utils.py:16-24."""
    h, w = image.shape[:2]
    side = max(h, w)
    pad = np.zeros((side, side, 3), dtype=np.uint8)
    top, left = int((side - h) // 2), int((side - w) // 2)
    pad[top:top + h, left:left + w] = image
    return pad, np.array([top, top + h, left, left + w, h, w], dtype=np.float32)


def img_preprocess(image, input_size=512):
    """utils.py:26-30 restated on the host with OpenCV exactly like the reference (BGR->RGB, square zero pad, cubic resize;
    returns uint8 [1,512,512,3]).  ``ROMP.forward`` does NOT use it - it runs ``ROMP.preprocess`` (one CUDA kernel); this
    host mirror exists for tests and for callers that batch pre-sized frames themselves."""
    import cv2
    image = cv2.cvtColor(image, cv2.COLOR_BGR2RGB)
    pad, info = padding_image(image)
    return cv2.resize(pad, (input_size, input_size), interpolation=cv2.INTER_CUBIC)[None], info


INVALID_TRANS = np.array([-1.0, -1.0, -1.0], np.float32)      # utils.py:295


def _translation_lsq_host(S, p2, focal, center):
    """estimate_translation_np (utils.py:347-389, the reference's own fallback), all joints valid, fp64 on the host."""
    n = S.shape[0]
    Z = np.reshape(np.tile(S[:, 2], (2, 1)).T, -1)
    XY = np.reshape(S[:, :2], -1)
    O_ = np.tile(center, n)
    Fv = np.tile(np.array([focal, focal], np.float64), n)
    w = np.ones(2 * n)
    Q = np.array([Fv * np.tile(np.array([1, 0]), n), Fv * np.tile(np.array([0, 1]), n), O_ - np.reshape(p2, -1)]).T
    c = (np.reshape(p2, -1) - O_) * Z - Fv * XY
    W = np.diagflat(w)
    Q, c = W @ Q, W @ c
    return np.linalg.solve(Q.T @ Q, Q.T @ c)


def estimate_translation_pnp(joints, cam, focal_length=443.4, img_size=512.0):
    """``--cam_trans pnp``: the reference's DEFAULT cam_trans (convert_cam_to_3d_trans2 post_parser.py:96-101 ->
    estimate_translation utils.py:391-436 -> estimate_translation_cv2 :331-345): per person
    cv2.solvePnPRansac(EPnP, reprojectionError 20, 100 iterations) on the 24 SMPL joints against their weak-perspective
    projection (pj2d + 1) * 256, K = diag(443.4) with principal point 256; INVALID_TRANS when RANSAC finds no inliers,
    the closed-form least squares (:347-389) when OpenCV raises.  Host side (OpenCV), like the reference; the device
    default (``--cam_trans lsq``) is that closed form for every person (b200romp_project)."""
    import cv2
    joints, cam = np.asarray(joints, np.float32), np.asarray(cam, np.float32)
    j3 = np.ascontiguousarray(joints[:, :24])
    p2 = (j3[:, :, :2] * cam[:, None, 0:1] + cam[:, None, 1:3] + 1.0) * (img_size / 2.0)      # batch_orth_proj utils.py:309-315
    K = np.eye(3)
    K[0, 0] = K[1, 1] = focal_length
    K[:2, 2] = img_size // 2
    out = np.zeros((len(j3), 3), np.float32)
    for i in range(len(j3)):
        try:
            _, _, tvec, inliers = cv2.solvePnPRansac(j3[i], p2[i].astype(np.float32), K, None, flags=cv2.SOLVEPNP_EPNP,
                                                     reprojectionError=20, iterationsCount=100)
            out[i] = INVALID_TRANS if inliers is None else tvec[:, 0]
        except Exception:
            out[i] = _translation_lsq_host(j3[i].astype(np.float64), p2[i].astype(np.float64), focal_length,
                                           np.array([img_size / 2.0, img_size / 2.0]))
    return out


def _ptr(t):
    return C.c_void_p(t.data_ptr())


class SMPLParser:
    """Seam S3 (post_parser.SMPL_parser, post_parser.py:116-125) on libb200romp's fused SMPL kernels."""

    def __init__(self, pack, device, n_betas=10, shape_key="shapedirs"):
        self.lib = _lib.load()
        g = lambda k, dt: np.ascontiguousarray(pack[k].detach().cpu().numpy() if isinstance(pack[k], torch.Tensor) else pack[k], dtype=dt)
        self._keep = [g("v_template", np.float32), g(shape_key, np.float32), g("posedirs", np.float32),
                      g("J_regressor", np.float32), g("weights", np.float32), g("kintree_table", np.int64),
                      g("extra_joints_index", np.int64), g("J_regressor_extra9", np.float32),
                      g("J_regressor_h36m17", np.float32)]
        k = self._keep
        assert k[0].shape == (6890, 3) and k[1].shape == (6890, 3, n_betas) and k[2].shape == (207, 20670)
        fp, lp = C.POINTER(C.c_float), C.POINTER(C.c_longlong)
        a = lambda x, t: x.ctypes.data_as(t)
        self.h = self.lib.b200romp_smpl_create(device, n_betas, a(k[0], fp), a(k[1], fp), a(k[2], fp), a(k[3], fp),
                                               a(k[4], fp), a(k[5], lp), a(k[6], lp), a(k[7], fp), a(k[8], fp))
        if not self.h:
            raise RuntimeError("b200romp_smpl_create: " + self.lib.b200romp_last_error().decode())
        self.n_betas = n_betas
        self.ws_floats = self.lib.b200romp_smpl_workspace_floats()
        self.faces = torch.from_numpy(np.ascontiguousarray(g("f", np.int64))) if "f" in pack else None

    def forward(self, betas, thetas, n, d_count, root_align, ws, verts, joints, stream):
        _lib.check(self.lib.b200romp_smpl_forward(self.h, _ptr(betas), betas.shape[1], _ptr(thetas), n,
                                                  None if d_count is None else _ptr(d_count), int(root_align),
                                                  _ptr(ws), _ptr(verts), _ptr(joints), C.c_void_p(stream)), "smpl_forward")

    def __del__(self):
        try:
            if getattr(self, "h", None):
                self.lib.b200romp_smpl_destroy(self.h)
        except Exception:
            pass


class MapsModule(torch.nn.Module):
    """``ROMP.model``: seam S1 as a module, like the reference's ``self.model`` (ROMPv1 wrapped in nn.DataParallel,
    main.py:74-77): ``model(frames)`` with frames [B,512,512,3] (uint8 / float32 0..255, device) returns
    ``(center_maps [B,1,64,64], params_maps [B,145,64,64])``.  Difference to the reference, by design: the cam-scale
    ``1.1**x`` of main.py:113 is already applied to ``params_maps[:,0]`` (it is fused into the head conv's epilogue)."""

    def __init__(self, owner):
        super().__init__()
        object.__setattr__(self, "_owner", owner)       # not a sub-module: no parameter / state-dict recursion

    def forward(self, frames):
        o = self._owner
        after_producers(o.stream, o.tdevice, frames)
        with torch.cuda.stream(o.stream):
            c, p = o.run_maps(frames.contiguous())
        torch.cuda.current_stream(o.tdevice).wait_stream(o.stream)
        return c, p


class ROMP(torch.nn.Module):
    """``ROMP(settings)(image_bgr)`` - same contract as simple_romp/romp/main.py:64-176."""

    def __init__(self, romp_settings, state_dict=None, smpl_pack=None):
        super().__init__()
        self.settings = s = romp_settings
        if not torch.cuda.is_available() or s.GPU < 0:
            raise RuntimeError("romp_b200.ROMP needs a CUDA device (H100, sm_90a); there is no CPU fallback")
        for flag in ("render_mesh", "show"):
            if getattr(s, flag, False):
                raise NotImplementedError(f"--{flag} is outside the GPU hot path (SURVEY.md section 2: out of scope)")
        if getattr(s, "onnx", False):
            raise NotImplementedError("--onnx: onnxruntime is not available offline; seam S1 is ROMP.model (MapsModule), the same "
                                      "seam the reference swaps for its ONNX session (main.py:78-91,108-110)")
        if getattr(s, "show_largest", False) and not getattr(s, "temporal_optimize", False):
            raise NotImplementedError("--show_largest only selects the smoothed person of --temporal_optimize (main.py:128-134)")
        self.video_streams = check_video_streams(s, bool(getattr(s, "temporal_optimize", False)))
        self.lib = _lib.load()
        self.device_index = int(s.GPU)
        self.tdevice = torch.device("cuda", self.device_index)
        torch.cuda.set_device(self.tdevice)
        self.precision = getattr(s, "precision", "bf16")
        self.max_batch = int(getattr(s, "max_batch", 64))
        if state_dict is None:
            state_dict = torch.load(s.model_path, map_location="cpu")          # main.py:75
        self._nets = {}
        self._state_dict = state_dict
        self.stream = torch.cuda.Stream(device=self.tdevice)
        self.calc_smpl = bool(s.calc_smpl)
        if self.calc_smpl:
            if smpl_pack is None:
                smpl_pack = torch.load(s.smpl_path, map_location="cpu")        # smpl.py:41
            self.smpl = SMPLParser(smpl_pack, self.device_index)
        self._alloc(self.max_batch)
        self.model = MapsModule(self)
        self.temporal = None
        if getattr(s, "temporal_optimize", False):                                 # main.py:117-125
            from .temporal import TemporalState
            self.temporal = TemporalState(bool(getattr(s, "show_largest", False)))
            self._tracks = self.lib.b200romp_tracks_create(self.device_index, self.temporal.n_slots)
            if not self._tracks:
                raise RuntimeError("b200romp_tracks_create: " + self.lib.b200romp_last_error().decode())
            self._slot_host = torch.zeros(self.cap, dtype=torch.int32).pin_memory()
            self._slot_dev = torch.zeros(self.cap, dtype=torch.int32, device=self.tdevice)
            # forward_video's device tracker: its own signals, tracks and filters (csrc/romp_track.cu); stream mode: one
            # independent tracker per signal_ID, which forward shares
            if self.video_streams:
                self._rtrack = self.lib.b200romp_romp_tracker_create_streams(self.device_index, self.video_streams)
            else:
                self._rtrack = self.lib.b200romp_romp_tracker_create(self.device_index, self.temporal.max_signals)
            if not self._rtrack:
                raise RuntimeError("b200romp_romp_tracker_create: " + self.lib.b200romp_last_error().decode())
            self._signal_codes = {}          # signal_ID -> int32 code of the device tracker (stream mode: stream index)
            self._temporal_user = None       # "forward" / "video": which path holds the tracker state

    # ------------------------------------------------------------------------------------------
    def _net(self, in_dtype):
        if in_dtype not in self._nets:
            build = graph.build_romp_resnet50 if getattr(self.settings, "backbone", "hrnet32") == "resnet50" else graph.build_romp
            self._nets[in_dtype] = build(self._state_dict, self.device_index, self.precision, in_dtype, self.max_batch)
        return self._nets[in_dtype]

    def _alloc(self, B):
        dev, cap = self.tdevice, B * MAX_PERSON
        f32, i64 = torch.float32, torch.int64
        self.cap = cap
        z = lambda *shape, dtype=f32: torch.zeros(*shape, dtype=dtype, device=dev)
        # shared scratch: only touched by kernels on self.stream, in order
        self.shared = dict(
            center_maps=z(B, 1, 64, 64), params_maps=z(B, N_PARAMS, 64, 64), flat_inds=z(cap, dtype=i64),
            params_pred=z(cap, N_PARAMS),
            parse_ws=torch.zeros(int(self.lib.b200romp_parse_workspace_bytes(B)), dtype=torch.uint8, device=dev))
        if self.calc_smpl:
            self.shared["smpl_ws"] = z(cap, self.smpl.ws_floats)
        # two slots of per-person outputs (+ pinned host mirrors) so that batch i+1 can be computed while batch i
        # is still being read back (forward_batches)
        self.slots = []
        for _ in range(2):
            d = dict(count=z(1, dtype=torch.int32), batch_ids=z(cap, dtype=i64), center_confs=z(cap, 1), cam=z(cap, 3),
                     thetas=z(cap, 72), betas=z(cap, 10), center_preds=z(cap, 2, dtype=i64), cam_trans=z(cap, 3),
                     pj2d_org=z(cap, 71, 2))
            if self.calc_smpl:
                d.update(verts=z(cap, 6890, 3), joints=z(cap, 71, 3))
            self.slots.append(dict(dev=d, host=None, count_host=torch.zeros(1, dtype=torch.int32).pin_memory(),
                                   done=torch.cuda.Event(), frames={}, h2d=torch.cuda.Event(),
                                   pad=z(B, 6), raw=RawStager(dev)))   # per-frame pad info, raw image staging
        self._slot = 0
        self.copy_stream = torch.cuda.Stream(device=dev)
        self.d2h_stream = torch.cuda.Stream(device=dev)

    @property
    def buf(self):
        """device buffers of the slot used by the most recent batch (+ the shared maps)"""
        return {**self.shared, **self.slots[self._slot]["dev"]}

    def _host(self, slot):
        if slot["host"] is None:      # pinned mirrors, allocated on first read-back
            slot["host"] = {k: torch.zeros(v.shape, dtype=v.dtype).pin_memory() for k, v in slot["dev"].items() if k != "count"}
        return slot["host"]

    # ------------------------------------------------------------------------------------------
    @torch.no_grad()
    def run_maps(self, frames_dev):
        """Seam S1 only: frames [B,512,512,3] uint8/float32 on the device -> (center_maps, params_maps) views."""
        B = frames_dev.shape[0]
        assert frames_dev.is_cuda and frames_dev.is_contiguous() and tuple(frames_dev.shape[1:]) == (512, 512, 3)
        assert B <= self.max_batch, f"batch {B} > max_batch {self.max_batch}"
        in_dtype = {torch.uint8: U8, torch.float32: F32}[frames_dev.dtype]
        nb, io = self._net(in_dtype)
        lib, sp = self.lib, C.c_void_p(self.stream.cuda_stream)
        _lib.check(lib.b200romp_net_bind(nb.net, io["frames"], _ptr(frames_dev)))
        _lib.check(lib.b200romp_net_bind(nb.net, io["center_maps"], _ptr(self.shared["center_maps"])))
        _lib.check(lib.b200romp_net_bind(nb.net, io["params_maps"], _ptr(self.shared["params_maps"])))
        _lib.check(lib.b200romp_net_run(nb.net, B, sp), "net_run")
        return self.shared["center_maps"][:B], self.shared["params_maps"][:B]

    @torch.no_grad()
    def run_parse(self, B, center_override=None, slot=None):
        """Seam S2 on the maps currently in the buffers (enqueued on self.stream, no host sync)."""
        sh, lib, sp = self.shared, self.lib, C.c_void_p(self.stream.cuda_stream)
        b = (self.slots[self._slot] if slot is None else slot)["dev"]
        center = sh["center_maps"] if center_override is None else center_override
        _lib.check(lib.b200romp_parse(_ptr(center), _ptr(sh["params_maps"]), B, 64, 10, float(self.settings.center_thresh),
                                      self.cap, _ptr(b["count"]), _ptr(b["batch_ids"]), _ptr(sh["flat_inds"]),
                                      _ptr(b["center_confs"]), _ptr(sh["params_pred"]), _ptr(b["cam"]), _ptr(b["thetas"]),
                                      _ptr(b["betas"]), _ptr(b["center_preds"]), _ptr(sh["parse_ws"]), sp), "parse")

    @torch.no_grad()
    def run_smpl_project(self, cap, offsets, slot=None, count_on_device=True, rows=None):
        """Seams S3-S4 for up to ``cap`` persons (the device-side count limits it further unless count_on_device=False).
        ``offsets``: one pad info [top,bottom,left,right,h,w] for every frame, or a device [B,6] table with one row per frame.
        ``rows``: the input rows (count, batch_ids, thetas, betas, cam) when they are not the slot's parse outputs."""
        sh, lib, sp = self.shared, self.lib, C.c_void_p(self.stream.cuda_stream)
        b = (self.slots[self._slot] if slot is None else slot)["dev"]
        r = b if rows is None else rows
        cnt = r["count"] if count_on_device else None
        cp = None if cnt is None else _ptr(cnt)
        per_frame = isinstance(offsets, torch.Tensor) and offsets.dim() == 2
        off = (C.c_float * 6)(*[float(v) for v in (FULL_FRAME if per_frame else offsets)])
        if self.calc_smpl:
            self.smpl.forward(r["betas"], r["thetas"], cap, cnt, self.settings.root_align, sh["smpl_ws"],
                              b["verts"], b["joints"], self.stream.cuda_stream)
            if per_frame:
                _lib.check(lib.b200romp_project_frames(_ptr(b["joints"]), None, _ptr(r["cam"]), cap, cp, _ptr(r["batch_ids"]),
                                                       _ptr(offsets), _ptr(b["pj2d_org"]), None, None, _ptr(b["cam_trans"]), sp),
                           "project_frames")
            else:
                _lib.check(lib.b200romp_project(_ptr(b["joints"]), None, _ptr(r["cam"]), cap, cp, off,
                                                _ptr(b["pj2d_org"]), None, None, _ptr(b["cam_trans"]), sp), "project")
            if getattr(self.settings, "cam_trans", "lsq") == "epnp":    # overwrites the closed form in place
                _lib.check(lib.b200romp_cam_trans_pnp(_ptr(b["joints"]), _ptr(r["cam"]), cap, cp, _ptr(b["cam_trans"]), None, sp),
                           "cam_trans_pnp")
        else:   # without SMPL the reference keeps the weak-perspective translation of main.py:166 (no pad info involved)
            _lib.check(lib.b200romp_project(_ptr(r["cam"]), None, _ptr(r["cam"]), cap, cp, off, None, None,
                                            _ptr(b["cam_trans"]), None, sp), "project")

    @torch.no_grad()
    def run_post(self, B, offsets, center_override=None, slot=None):
        """Seams S2-S4 on the maps currently in the buffers; everything enqueued on self.stream, no host sync."""
        self.run_parse(B, center_override, slot)
        self.run_smpl_project(B * MAX_PERSON, offsets, slot)

    def _views(self, src, n):
        out = {"cam": src["cam"][:n], "global_orient": src["thetas"][:n, :3], "body_pose": src["thetas"][:n, 3:],
               "smpl_betas": src["betas"][:n], "smpl_thetas": src["thetas"][:n], "center_preds": src["center_preds"][:n],
               "center_confs": src["center_confs"][:n], "cam_trans": src["cam_trans"][:n]}
        if self.calc_smpl:
            out.update(verts=src["verts"][:n], joints=src["joints"][:n], pj2d_org=src["pj2d_org"][:n])
        out["pred_batch_ids"] = src["batch_ids"][:n]
        return out

    def record_layout(self):
        """Fixed per-person record of this configuration for the sharded path's single all-gather (shard.ShardGather)."""
        from . import shard
        return shard.romp_layout(self.calc_smpl, 10)

    def record_fields(self, slot=None):
        """name -> device tensor [cap, ...] of the slot used by the most recent batch, keyed like record_layout()."""
        d = (self.slots[self._slot] if slot is None else slot)["dev"]
        f = {"cam": d["cam"], "smpl_thetas": d["thetas"], "smpl_betas": d["betas"], "center_confs": d["center_confs"],
             "cam_trans": d["cam_trans"], "center_preds": d["center_preds"], "pred_batch_ids": d["batch_ids"]}
        if self.calc_smpl:
            f.update(joints=d["joints"], pj2d_org=d["pj2d_org"], verts=d["verts"])
        return f, d["count"]

    def collect(self, to_numpy=True, slot=None, stream=None):
        """The single host sync of a batch: person count, then D2H of the N valid rows (utils.py:32-41) into pinned
        host mirrors.  The returned numpy arrays are views of those mirrors: valid until the slot is reused, i.e.
        until the second-next batch (copy them if they must live longer)."""
        slot = self.slots[self._slot] if slot is None else slot
        stream = self.stream if stream is None else stream
        with torch.cuda.stream(stream):
            slot["count_host"].copy_(slot["dev"]["count"], non_blocking=True)
        stream.synchronize()
        n = int(slot["count_host"].item())
        if n == 0:
            return None
        if not to_numpy:
            return self._views(slot["dev"], n)
        host = self._host(slot)
        with torch.cuda.stream(stream):
            for k, v in slot["dev"].items():
                if k != "count":
                    host[k][:n].copy_(v[:n], non_blocking=True)
        stream.synchronize()
        return {k: v.numpy() for k, v in self._views(host, n).items()}

    # ------------------------------------------------------------------------------------------
    def _apply_cam_trans(self, out):
        """``--cam_trans pnp``: the reference's default estimator replaces the device's closed form, on the host."""
        if getattr(self.settings, "cam_trans", "lsq") == "pnp" and self.calc_smpl:
            out["cam_trans"] = estimate_translation_pnp(out["joints"], out["cam"])
        return out

    @torch.no_grad()
    def forward_batch(self, frames, offsets=None, to_numpy=True, center_override=None, own=True):
        """frames: [B,512,512,3] RGB uint8/float32 (torch tensor, pinned host or device, or numpy), already
        padded+resized like img_preprocess.  Returns the reference's dict plus ``pred_batch_ids`` or None.
        ``offsets``: the pad info [top,bottom,left,right,h,w] of every frame, or one row per frame ([B,6], numpy or
        tensor) when the frames come from images of different sizes.
        Device-resident ``frames`` / ``center_override`` / ``offsets`` may come straight from a producer on the caller's
        current stream.  ``own=True`` (default) returns arrays that own their memory; ``own=False`` returns views of the
        pinned read-back mirrors, valid until the second-next batch.  ``to_numpy=False`` returns device tensors of the
        caller's current stream (see forward_batches)."""
        after_producers(self.stream, self.tdevice, center_override, offsets)
        out = self._result(self._submit_frames(frames, offsets, center_override), to_numpy)
        if out is not None and to_numpy and own:
            out = self._apply_cam_trans({k: np.array(v) for k, v in out.items()})
        return out

    @torch.no_grad()
    def forward_batches(self, batches, offsets=None, center_override=None, to_numpy=True, gather=None, frame_offset=0):
        """Pipelined streaming over an iterable of frame batches (video): yields one result dict (or None) per batch,
        in order.  H2D of batch i+1 (copy stream) and D2H of batch i-1 (read-back stream) overlap the kernels of
        batch i; the host waits only for the H2D copy of the batch it just handed over and for the person count of an
        already finished batch.  Stream-order contract:
        - a host batch has been copied when the generator pulls the next one, so a caller may refill one (pinned or
          numpy) buffer in place in its decode loop;
        - device-resident frames, ``center_override`` and per-frame ``offsets`` may come from producers on the caller's
          current stream (the model's streams wait for it) and may be dropped right after they are handed over;
        - with ``to_numpy=True`` the yielded arrays are views of pinned mirrors: they hold batch i until the generator
          is resumed for batch i+2, whose read-back reuses them;
        - with ``to_numpy=False`` the yielded tensors are copies made on the caller's current stream after the batch's
          kernels: the caller may read them there at any later time, and the model's kernels wait for the copies
          before they reuse the slot.
        Sharded (multi-GPU) use: pass ``gather`` (a shard.ShardGather built on ``record_layout()``) and this rank's
        ``frame_offset``; each batch's records are then packed and all-gathered on the gather's side stream right after
        its kernels, and the generator yields ``(own_result, gather_handle)`` pairs (own shard read back to this rank's
        host; ``gather.result(handle)`` gives every rank's persons on the device)."""
        pending = None
        after_producers(self.stream, self.tdevice, center_override, offsets)
        for frames in batches:
            slot = self._submit_frames(frames, offsets, center_override, gather, frame_offset)
            if pending is not None:
                res = self._result(pending, to_numpy)
                yield (res, pending["gather"]) if gather is not None else res
            pending = slot
        if pending is not None:
            res = self._result(pending, to_numpy)
            yield (res, pending["gather"]) if gather is not None else res

    def _submit_frames(self, frames, offsets, center_override, gather=None, frame_offset=0):
        """One batch of frames into the next slot: H2D into the slot's frame buffer on the copy stream, the kernels on
        self.stream.  Returns once host frames have been copied, so the caller may refill their buffer."""
        if isinstance(frames, np.ndarray):
            frames = torch.from_numpy(frames)
        B = frames.shape[0]
        self._slot ^= 1
        slot = self.slots[self._slot]
        fd = frame_buffer(slot["frames"], frames.dtype, B, self.tdevice)
        after_producers(self.copy_stream, self.tdevice, frames)
        with torch.cuda.stream(self.copy_stream):
            self.copy_stream.wait_event(slot["done"])          # the slot's previous kernels no longer read fd
            fd.copy_(frames, non_blocking=True)
            slot["h2d"].record(self.copy_stream)
        with torch.cuda.stream(self.stream):
            self.stream.wait_event(slot["h2d"])
            if slot.get("packed") is not None:
                self.stream.wait_event(slot["packed"])          # the gather's pack kernel has read the slot's previous results
            self.run_maps(fd)
            self.run_post(B, frame_offsets(offsets, slot["pad"], B), center_override, slot)
            slot["done"].record(self.stream)
            if gather is not None:
                fields, count = self.record_fields(slot)
                slot["gather"] = gather.submit(fields, count, frame_offset)
                slot["packed"] = slot["gather"]["packed"]
        if not frames.is_cuda:
            slot["h2d"].synchronize()     # the caller may refill its (single) host buffer as soon as we yield / pull the next batch
        return slot

    def _read_back(self, slot, to_numpy=True):
        self.d2h_stream.wait_event(slot["done"])
        return self.collect(to_numpy, slot, self.d2h_stream)   # device views stay valid until the slot's next batch

    def _result(self, slot, to_numpy):
        """A batch's result for the caller: arrays (to_numpy), else copies of the slot's rows on the caller's stream."""
        out = self._read_back(slot, to_numpy)
        return out if out is None or to_numpy else to_caller([out], slot["done"], self.stream)[0]

    @torch.no_grad()
    def forward_images(self, images, to_numpy=True, center_override=None):
        """Batched ``forward`` on raw images of any sizes: ``images`` is a sequence of HxWx3 uint8 BGR images (numpy arrays,
        host or device tensors), run in chunks of at most ``max_batch``.  Returns a list of the same length whose element
        i is what ``forward(images[i])`` returns (the reference's dict without ``pred_batch_ids``, or None; nothing is
        printed).  center_override: optional device [n,1,64,64] replacing the images' center maps (tests, measurement)."""
        return next(self.forward_image_batches([images], to_numpy, center_override))

    @torch.no_grad()
    def forward_image_batches(self, batches, to_numpy=True, center_override=None):
        """Streaming form of ``forward_images`` over an iterable of image lists: yields one result list per input list, in
        order.  Each chunk of at most ``max_batch`` images is staged into its slot's pinned buffer and sent with one H2D
        on the copy stream (device images are read in place), preprocessed by one kernel into the slot's frames with
        a per-frame pad table, and post-processed with each frame's own geometry; staging chunk i+1 and reading back
        chunk i-1 overlap the kernels of chunk i (the two slots of ``forward_batches``).  center_override applies to
        every list, entry k to the k-th image of the list.  Host images have been staged when the generator pulls the
        next list; device images and ``center_override`` may come from producers on the caller's current stream.  The
        yielded results own their memory: arrays, or with ``to_numpy=False`` device tensors copied on the caller's
        current stream (as in ``forward_batches``)."""
        if self.temporal is not None:
            raise NotImplementedError("--temporal_optimize smooths one image sequence: call forward_video() (or forward() per frame)")
        after_producers(self.stream, self.tdevice, center_override)

        def chunks():
            for images in batches:
                imgs = [image_tensor(x) for x in images]
                res = [None] * len(imgs)
                if not imgs:
                    yield res, imgs, 0, True
                for c0 in range(0, len(imgs), self.max_batch):
                    yield res, imgs[c0:c0 + self.max_batch], c0, c0 + self.max_batch >= len(imgs)

        pending = None
        for res, imgs, c0, last in chunks():
            co = None if center_override is None else center_override[c0:c0 + len(imgs)]
            slot = self._submit_images(imgs, co) if imgs else None
            if pending is not None:
                done = self._finish_images(*pending, to_numpy)
                if done is not None:
                    yield done
            pending = (slot, res, c0, len(imgs), last)
        if pending is not None:
            yield self._finish_images(*pending, to_numpy)

    def _upload(self, slot, imgs):
        """Host images into the slot's pinned staging buffer and to the device with one H2D on the copy stream; self.stream
        is ordered after that copy and after the producers of device images.  Returns each image's byte offset in
        slot["raw"].dev (None: a device image, read in place)."""
        raw = slot["raw"]
        offs, total = raw.stage(imgs, replace_after=slot["done"], reuse_after=slot["h2d"])
        if total:
            with torch.cuda.stream(self.copy_stream):
                self.copy_stream.wait_event(slot["done"])  # the slot's previous preprocessing no longer reads raw.dev
                raw.upload(total)
                slot["h2d"].record(self.copy_stream)
            self.stream.wait_event(slot["h2d"])
        after_producers(self.stream, self.tdevice, *imgs)
        return offs

    def _preprocess_images(self, imgs):
        """Raw images into the next slot's frames and pad table: one preprocessing kernel on self.stream."""
        self._slot ^= 1
        slot = self.slots[self._slot]
        fd = frame_buffer(slot["frames"], torch.uint8, len(imgs), self.tdevice)
        offs = self._upload(slot, imgs)
        with torch.cuda.stream(self.stream):
            preprocess_bgr_batch(self.lib, imgs, offs, slot["raw"].dev, fd, slot["pad"], self.stream.cuda_stream)
        return slot, fd

    def _submit_images(self, imgs, center_override):
        B = len(imgs)
        slot, fd = self._preprocess_images(imgs)
        with torch.cuda.stream(self.stream):
            self.run_maps(fd)
            self.run_post(B, slot["pad"][:B], center_override, slot)
            slot["done"].record(self.stream)
        return slot

    def _finish_images(self, slot, res, c0, B, last, to_numpy):
        """Read back one chunk and scatter its persons to res[c0:c0+B]; returns res once its last chunk is in."""
        out = None if slot is None else self._read_back(slot, to_numpy)
        if out is not None:
            with torch.cuda.stream(self.d2h_stream):        # device frame ids are read after the slot's kernels
                frames = split_by_frame(out, B, to_numpy)
            if not to_numpy:
                frames = to_caller(frames, slot["done"], self.stream)
            for i, r in enumerate(frames):
                if len(r["cam"]):
                    r.pop("pred_batch_ids")
                    res[c0 + i] = self._apply_cam_trans(r) if to_numpy else r
        return res if last else None

    @torch.no_grad()
    def preprocess(self, image, out=None):
        """img_preprocess (utils.py:26-30) on the GPU: raw HxWx3 uint8 BGR image (numpy / host tensor / device tensor) ->
        ``out`` [512,512,3] uint8 RGB on the device (allocated when None) + pad info [top,bottom,left,right,h,w].
        One kernel (b200romp_preprocess_bgr) on self.stream; a host image is staged through the current slot."""
        img = image_tensor(image)
        h, w = int(img.shape[0]), int(img.shape[1])
        if out is None:
            out = torch.empty((512, 512, 3), dtype=torch.uint8, device=self.tdevice)
        slot = self.slots[self._slot]
        off = self._upload(slot, [img])[0]
        raw, stride = (img.data_ptr(), img.stride(0)) if off is None else (slot["raw"].dev.data_ptr() + off, 3 * w)
        pad = (C.c_float * 6)()
        _lib.check(self.lib.b200romp_preprocess_bgr(C.c_void_p(raw), h, w, stride, 512, _ptr(out), pad,
                                                    C.c_void_p(self.stream.cuda_stream)), "preprocess_bgr")
        slot["done"].record(self.stream)                  # the slot's staging buffer is read until here
        return out, np.array(list(pad), dtype=np.float32)

    @torch.no_grad()
    def forward(self, image, signal_ID=0, **kwargs):
        """image: HxWx3 uint8 BGR (cv2.imread).  main.py:160-176; preprocessing, model, parse, SMPL and projection all run
        on the GPU - OpenCV is not involved."""
        if self.temporal is not None and self.video_streams:     # stream mode: one state for forward and forward_video
            out = self.forward_video([image], [signal_ID])[0]
            if out is None:
                print("None person detected")
            return out
        if self.temporal is not None:
            self._claim_temporal("forward")
            return self._forward_temporal(image, signal_ID)
        out = self.forward_images([image])[0]
        if out is None:
            print("None person detected")                                       # post_parser.py:139
        return out

    @torch.no_grad()
    def _forward_temporal(self, image, signal_ID):
        """forward() with --temporal_optimize (main.py:164-165 -> temporal_optimization :127-157): parse, associate the
        detections with tracks on the host (needs the cams: one small D2H, like the reference), One-Euro smoothing of
        thetas / betas / cam on the device, then SMPL + projection on the smoothed parameters."""
        slot, fd = self._preprocess_images([image_tensor(image)])
        b, lib, sp = slot["dev"], self.lib, C.c_void_p(self.stream.cuda_stream)
        with torch.cuda.stream(self.stream):
            self.run_maps(fd)
            self.run_parse(1, None, slot)
            slot["count_host"].copy_(b["count"], non_blocking=True)
        self.stream.synchronize()
        n = int(slot["count_host"].item())
        if n == 0:
            print("None person detected")
            return None
        with torch.cuda.stream(self.stream):
            cams = b["cam"][:n].cpu().numpy()
            raw_thetas = b["thetas"][:n].clone()          # global_orient / body_pose keep the UNsmoothed values (main.py:148-153)
        slots, track_ids, reset = self.temporal.assign(cams, signal_ID)
        for sl in reset:
            _lib.check(lib.b200romp_tracks_reset(self._tracks, int(sl), sp), "tracks_reset")
        self._slot_host[:n].copy_(torch.from_numpy(slots))
        n_smpl = n
        with torch.cuda.stream(self.stream):
            self._slot_dev[:n].copy_(self._slot_host[:n], non_blocking=True)
            _lib.check(lib.b200romp_one_euro_smooth(self._tracks, _ptr(self._slot_dev), n, None, _ptr(b["thetas"]), _ptr(b["betas"]),
                                                    10, 10, _ptr(b["cam"]), float(self.settings.smooth_coeff), 30.0,
                                                    int(not self.temporal.show_largest), sp), "one_euro")
            if self.temporal.show_largest:                 # only the largest person goes on (main.py:129-134)
                k = int(np.argmax(cams[:, 0]))
                for key in ("thetas", "betas", "cam"):
                    b[key][0].copy_(b[key][k].clone())
                n_smpl = 1
            self.run_smpl_project(n_smpl, slot["pad"][:1], slot, count_on_device=False)
            slot["done"].record(self.stream)
            host = self._host(slot)
            for key, v in b.items():
                if key != "count":
                    host[key][:n].copy_(v[:n], non_blocking=True)
            raw_host = raw_thetas.cpu()
        self.stream.synchronize()
        v = {k: np.array(t.numpy()) for k, t in self._views(host, n).items()}
        v.pop("pred_batch_ids")
        v["global_orient"], v["body_pose"] = raw_host.numpy()[:, :3].copy(), raw_host.numpy()[:, 3:].copy()
        for key in ("smpl_thetas", "smpl_betas", "cam", "cam_trans", "verts", "joints", "pj2d_org"):
            if key in v:
                v[key] = v[key][:n_smpl]
        if track_ids is not None:
            v["track_ids"] = track_ids                      # main.py:156
        return v

    # ------------------------------------------------------------------------------------------
    # video mode in batches (-t/--temporal_optimize): the per-frame temporal path of forward, on the batched image path
    def _claim_temporal(self, user):
        """forward and forward_video keep separate tracker state: one of them per video (reset_temporal() between)."""
        if self._temporal_user not in (None, user):
            raise RuntimeError(f"--temporal_optimize: this instance's video is being run by {self._temporal_user}(); call "
                               f"reset_temporal() before switching to {user}()")
        self._temporal_user = user

    def reset_temporal(self, signal_ID=None):
        """Start a new video: forget every signal, track id and filter of both forward() and forward_video(); ids count
        from 1 again.  Stream mode (--video_streams) with a ``signal_ID``: forget that stream only (its index is freed;
        when the signal_ID comes back its ids start at 1)."""
        if self.temporal is None:
            raise RuntimeError("reset_temporal: this ROMP instance was built without -t/--temporal_optimize")
        if signal_ID is not None:
            if not self.video_streams:
                raise ValueError("reset_temporal(signal_ID): only in stream mode (--video_streams)")
            self._signal_codes.pop(signal_ID, None)    # the index is reset when a signal_ID takes it again
            return
        from .temporal import TemporalState
        sp = C.c_void_p(self.stream.cuda_stream)
        self.temporal = TemporalState(self.temporal.show_largest, self.temporal.max_signals)
        _lib.check(self.lib.b200romp_tracks_reset(self._tracks, -1, sp), "tracks_reset")
        _lib.check(self.lib.b200romp_romp_tracker_reset(self._rtrack, sp), "romp_tracker_reset")
        self._signal_codes = {}
        self._temporal_user = None

    def _reset_stream(self, k):
        """Stream mode: stream index k starts afresh, on the model's stream (before the next track step)."""
        _lib.check(self.lib.b200romp_romp_tracker_reset_stream(self._rtrack, k, C.c_void_p(self.stream.cuda_stream)),
                   "romp_tracker_reset_stream")

    def _video_buffers(self, slot):
        """The track step's outputs of one slot (allocated on first use): the smoothed rows SMPL runs on, the per-row
        filter slot and track id, the frames' signal codes and pinned read-back mirrors."""
        if "video" not in slot:
            dev, cap, B = self.tdevice, self.cap, self.max_batch
            z = lambda *shape, dtype=torch.float32: torch.zeros(*shape, dtype=dtype, device=dev)
            slot["video"] = dict(count=z(1, dtype=torch.int32), batch_ids=z(cap, dtype=torch.int64), thetas=z(cap, 72),
                                 betas=z(cap, 10), cam=z(cap, 3), slot=z(cap, dtype=torch.int32), track_ids=z(cap, dtype=torch.int32),
                                 codes=z(B, dtype=torch.int32), codes_host=torch.zeros(B, dtype=torch.int32).pin_memory(),
                                 codes_h2d=torch.cuda.Event(), counts_host=torch.zeros(2, dtype=torch.int32).pin_memory(), host=None)
        return slot["video"]

    def run_track_step(self, B, codes, slot):
        """The video mode's association and One-Euro smoothing of a chunk's B frames (b200romp_romp_track_step), enqueued
        on self.stream after the parse: no host sync.  ``codes``: the int32 signal code of every frame."""
        v = self._video_buffers(slot)
        v["codes_h2d"].synchronize()               # the pinned codes of the slot's previous chunk have been copied
        v["codes_host"][:B].copy_(torch.as_tensor(codes, dtype=torch.int32))
        b, s = slot["dev"], self.settings
        with torch.cuda.stream(self.stream):
            v["codes"][:B].copy_(v["codes_host"][:B], non_blocking=True)
            v["codes_h2d"].record(self.stream)
            _lib.check(self.lib.b200romp_romp_track_step(
                self._rtrack, B, self.cap, _ptr(b["count"]), _ptr(b["batch_ids"]), _ptr(b["cam"]), _ptr(b["thetas"]),
                _ptr(b["betas"]), _ptr(v["codes"]), int(self.temporal.show_largest), float(s.smooth_coeff), 30.0, _ptr(v["count"]),
                _ptr(v["batch_ids"]), _ptr(v["thetas"]), _ptr(v["betas"]), _ptr(v["cam"]), _ptr(v["slot"]), _ptr(v["track_ids"]),
                C.c_void_p(self.stream.cuda_stream)), "romp_track_step")
        return v

    def _submit_video(self, imgs, codes, center_override):
        B = len(imgs)
        slot, fd = self._preprocess_images(imgs)
        with torch.cuda.stream(self.stream):
            self.run_maps(fd)
            self.run_parse(B, center_override, slot)
            v = self.run_track_step(B, codes, slot)
            # tracked: every row (count on the device); --show_largest: the chunk's <= B compacted largest rows
            self.run_smpl_project(B if self.temporal.show_largest else B * MAX_PERSON, slot["pad"][:B], slot, rows=v)
            slot["done"].record(self.stream)
        return slot

    def _read_back_video(self, slot, B, to_numpy):
        """The chunk's one host sync (both row counts), then its rows -> one result per frame, like forward()."""
        st, v, d = self.d2h_stream, slot["video"], slot["dev"]
        st.wait_event(slot["done"])
        with torch.cuda.stream(st):
            v["counts_host"][0:1].copy_(d["count"], non_blocking=True)
            v["counts_host"][1:2].copy_(v["count"], non_blocking=True)
        st.synchronize()
        n, m = int(v["counts_host"][0]), int(v["counts_host"][1])
        res = [None] * B
        if n == 0:
            return res
        tracked = not self.temporal.show_largest
        per = dict(center_preds=d["center_preds"], center_confs=d["center_confs"], raw=d["thetas"], ids=d["batch_ids"])
        if tracked:
            per["track_ids"] = v["track_ids"]
        rows = dict(cam=v["cam"], smpl_thetas=v["thetas"], smpl_betas=v["betas"], cam_trans=d["cam_trans"], ids=v["batch_ids"])
        if self.calc_smpl:
            rows.update(verts=d["verts"], joints=d["joints"], pj2d_org=d["pj2d_org"])
        if to_numpy:
            if v["host"] is None:
                v["host"] = {k: torch.zeros(t.shape, dtype=t.dtype).pin_memory() for k, t in
                             [("p_" + k, t) for k, t in per.items()] + [("r_" + k, t) for k, t in rows.items()]}
            h = v["host"]
            with torch.cuda.stream(st):
                for k, t in per.items():
                    h["p_" + k][:n].copy_(t[:n], non_blocking=True)
                for k, t in rows.items():
                    h["r_" + k][:m].copy_(t[:m], non_blocking=True)
            st.synchronize()
            per = {k: h["p_" + k][:n].numpy() for k in per}
            rows = {k: h["r_" + k][:m].numpy() for k in rows}
            own = np.array
        else:
            per = {k: t[:n] for k, t in per.items()}
            rows = {k: t[:m] for k, t in rows.items()}
            own = lambda t: t                                # views, copied for the caller by to_caller below
        ids = lambda t: t.cpu().numpy() if isinstance(t, torch.Tensor) else t
        with torch.cuda.stream(st):                          # device frame ids are read after the slot's kernels
            pb = np.searchsorted(ids(per["ids"]), np.arange(B + 1)).tolist()
            rb = np.searchsorted(ids(rows["ids"]), np.arange(B + 1)).tolist()
        for i in range(B):
            s, e, a, z = pb[i], pb[i + 1], rb[i], rb[i + 1]
            if s == e:
                continue
            r = {k: own(rows[k][a:z]) for k in rows if k != "ids"}
            r.update(global_orient=own(per["raw"][s:e, :3]), body_pose=own(per["raw"][s:e, 3:]),
                     center_preds=own(per["center_preds"][s:e]), center_confs=own(per["center_confs"][s:e]))
            if tracked:
                r["track_ids"] = own(per["track_ids"][s:e])
            res[i] = r
        return res if to_numpy else to_caller(res, slot["done"], self.stream)

    @torch.no_grad()
    def forward_video(self, images, signal_IDs=None, to_numpy=True, center_override=None):
        """Video mode (-t/--temporal_optimize) in batches: ``images`` (HxWx3 uint8 BGR, any sizes, numpy or host / device
        tensors) are consecutive frames, run in chunks of at most ``max_batch`` through the batched image path, with the
        association and One-Euro smoothing of every chunk as one kernel between the parse and SMPL (one host sync per
        chunk).  ``signal_IDs``: one per image (default 0).  Element i of the result is what ``forward(images[i],
        signal_IDs[i])`` returns in a loop on a fresh instance, or None; nothing is printed.  Like forward's temporal path
        it keeps the device's cam_trans: the closed form, or ``--cam_trans epnp`` on the smoothed rows (``--cam_trans pnp``,
        a host step, is not applied).  center_override: optional device
        [n,1,64,64] replacing the images' center maps (tests, measurement).  With --video_streams every signal_ID is an
        independent video (its own tracker, ids from 1 and filters, romp_b200/streams.py), stepped in parallel."""
        sids = None if signal_IDs is None else [signal_IDs]
        return next(self.forward_video_batches([images], sids, to_numpy, center_override))

    @torch.no_grad()
    def forward_video_batches(self, batches, signal_IDs=None, to_numpy=True, center_override=None):
        """Streaming form of ``forward_video`` over an iterable of image lists (consecutive parts of one video; the tracker
        state carries across lists): yields one result list per input list, in order, on forward_image_batches' two-slot
        pipeline.  ``signal_IDs``: None (every frame signal 0) or an iterable with one sequence of signal IDs per list.
        center_override applies to every list, entry k to the k-th image of the list.  Inputs and results follow
        ``forward_image_batches``: results own their memory (``to_numpy=False``: device copies on the caller's stream)."""
        if self.temporal is None:
            raise RuntimeError("forward_video needs -t/--temporal_optimize")
        after_producers(self.stream, self.tdevice, center_override)
        sid_iter = None if signal_IDs is None else iter(signal_IDs)

        def chunks():
            for images in batches:
                imgs = [image_tensor(x) for x in images]
                sids = [0] * len(imgs) if sid_iter is None else list(next(sid_iter))
                if len(sids) != len(imgs):
                    raise ValueError(f"forward_video: {len(sids)} signal_IDs for {len(imgs)} images")
                self._claim_temporal("video")
                if self.video_streams:
                    codes = stream_indices(self._signal_codes, sids, self.video_streams, self._reset_stream)
                else:
                    codes = [self._signal_codes.setdefault(sid, len(self._signal_codes)) for sid in sids]
                res = [None] * len(imgs)
                if not imgs:
                    yield res, imgs, codes, 0, True
                for c0 in range(0, len(imgs), self.max_batch):
                    yield res, imgs[c0:c0 + self.max_batch], codes[c0:c0 + self.max_batch], c0, c0 + self.max_batch >= len(imgs)

        pending = None
        for res, imgs, codes, c0, last in chunks():
            co = None if center_override is None else center_override[c0:c0 + len(imgs)]
            slot = self._submit_video(imgs, codes, co) if imgs else None
            if pending is not None:
                done = self._finish_video(*pending, to_numpy)
                if done is not None:
                    yield done
            pending = (slot, res, c0, len(imgs), last)
        if pending is not None:
            yield self._finish_video(*pending, to_numpy)

    def _finish_video(self, slot, res, c0, B, last, to_numpy):
        if slot is not None:
            res[c0:c0 + B] = self._read_back_video(slot, B, to_numpy)
        return res if last else None

    def __del__(self):
        try:
            if getattr(self, "_tracks", None):
                self.lib.b200romp_tracks_destroy(self._tracks)
            if getattr(self, "_rtrack", None):
                self.lib.b200romp_romp_tracker_destroy(self._rtrack)
        except Exception:
            pass


default_settings = None   # the reference evaluates romp_settings([]) at import (main.py:62); we do not


def check_cli(args):
    """What the ``romp`` command line refuses, before a model is built: display and rendering (with the messages of
    ``ROMP``), and any mode but image and video (webcam capture is not provided)."""
    for flag in ("render_mesh", "show"):
        if getattr(args, flag, False):
            raise NotImplementedError(f"--{flag} is outside the GPU hot path (SURVEY.md section 2: out of scope)")
    if args.mode not in ("image", "video"):
        raise NotImplementedError("video/webcam loops are outside the hot path; call ROMP.forward per frame")
    from .cli import check_inputs
    check_inputs(args)


def main(input_args=None):
    """The ``romp`` command (main.py:178-196).  ``--mode image`` writes ``<save_path>/<input stem>.npz`` when somebody
    is detected; ``--mode video`` writes the reference's per-frame PNG and npz files, ``video_results.npz`` and with
    ``--save_video`` the mp4 (romp_b200/cli.py), for ``-i`` or for each of ``--inputs``."""
    import cv2
    args = romp_settings(sys.argv[1:] if input_args is None else input_args)
    check_cli(args)
    romp = ROMP(args)
    if args.mode == "video":
        from . import cli
        if args.inputs is not None:
            cli.run_inputs_command(romp, args)
        else:
            cli.run_video(romp, args)
        return
    outputs = romp(cv2.imread(args.input))
    if outputs is not None:
        os.makedirs(args.save_path, exist_ok=True)
        np.savez(osp.join(args.save_path, osp.splitext(osp.basename(args.input))[0] + ".npz"), results=outputs)


if __name__ == "__main__":
    main()
