"""Host staging shared by ROMP and BEV: raw images and 512x512 frames on their way to the device, and the stream
ordering of device inputs.  Python here only moves bytes; the preprocessing is one CUDA kernel."""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _lib

FULL_FRAME = [0, 512, 0, 512, 512, 512]      # pad info of a frame that is already 512x512


def image_tensor(image):
    """HxWx3 uint8 BGR image (numpy, host or device tensor) -> a torch tensor the batched preprocessing can read: host
    images as they are (they are copied into pinned staging), device images in place when their rows are packed BGR
    pixels (any row stride >= 3w), else a contiguous copy."""
    t = torch.from_numpy(np.ascontiguousarray(image)) if isinstance(image, np.ndarray) else image
    assert isinstance(t, torch.Tensor) and t.dtype == torch.uint8 and t.dim() == 3 and t.shape[2] == 3, "image must be HxWx3 uint8 (BGR)"
    assert t.shape[0] > 0 and t.shape[1] > 0, "empty image"
    if t.is_cuda and not (t.stride(2) == 1 and t.stride(1) == 3 and t.stride(0) >= 3 * t.shape[1]):
        t = t.contiguous()
    return t


def staging_layout(images):
    """Byte offset of every host image inside one staging buffer (256-byte aligned; None for device images) and its size."""
    offs, total = [], 0
    for t in images:
        offs.append(None if t.is_cuda else total)
        if not t.is_cuda:
            total += (t.numel() + 255) // 256 * 256
    return offs, total


def stage_host_images(images, offs, raw_host):
    """Copy the host images into the pinned staging buffer (torch's copy_ splits each large copy over its CPU threads)."""
    for t, o in zip(images, offs):
        if o is not None:
            raw_host[o:o + t.numel()].view(t.shape).copy_(t)


def preprocess_bgr_batch(lib, images, offs, raw_dev, out, pad_table, stream):
    """b200romp_preprocess_bgr_batch: images[i] (device tensor, or host tensor staged at raw_dev[offs[i]:]) -> out[i]
    [512,512,3] uint8 RGB on the device, pad info into the device table pad_table [n,6] (may be None)."""
    n = len(images)
    ptrs = [t.data_ptr() if o is None else raw_dev.data_ptr() + o for t, o in zip(images, offs)]
    strides = [t.stride(0) if o is None else 3 * int(t.shape[1]) for t, o in zip(images, offs)]
    _lib.check(lib.b200romp_preprocess_bgr_batch((C.c_void_p * n)(*ptrs), (C.c_int * n)(*[int(t.shape[0]) for t in images]),
                                                 (C.c_int * n)(*[int(t.shape[1]) for t in images]), (C.c_int * n)(*strides), n, 512,
                                                 C.c_void_p(out.data_ptr()),
                                                 None if pad_table is None else C.c_void_p(pad_table.data_ptr()), C.c_void_p(stream)),
               "preprocess_bgr_batch")


def split_by_frame(out, n_frames, to_numpy):
    """A batch result whose rows come in frame order -> one dict per frame with that frame's rows of every field
    (possibly none): arrays that own their memory (to_numpy) or device views of ``out`` (for to_caller).  Device frame
    ids are read on the current stream."""
    ids = out["pred_batch_ids"]
    ids = ids.cpu().numpy() if isinstance(ids, torch.Tensor) else ids
    b = np.searchsorted(np.asarray(ids), np.arange(n_frames + 1)).tolist()
    return [{k: (np.array(v[s:e]) if to_numpy else v[s:e]) for k, v in out.items()} for s, e in zip(b[:-1], b[1:])]


def to_caller(results, done, stream):
    """Device results (``to_numpy=False``) handed to the caller: ``results`` is a list of dicts of device views of a
    slot's rows (or None), the slot's kernels end at the event ``done``, and ``stream`` writes the slot's next batch.
    Returns copies made on the caller's current stream after ``done``, so that they belong to that stream like any
    tensor the caller allocates there (the allocator recycles them in its order, not in the read-back's), and makes
    ``stream`` wait for the copies before it overwrites the slot.  No host sync."""
    cur = torch.cuda.current_stream(stream.device)
    cur.wait_event(done)
    out = [None if r is None else {k: v.clone() for k, v in r.items()} for r in results]
    stream.wait_stream(cur)
    return out


def after_producers(stream, device, *tensors):
    """Device-resident inputs were produced on the caller's current stream and ``stream`` reads them.  Order ``stream``
    after the caller's stream (once, no host sync) and keep the allocator from recycling the inputs while ``stream``
    still reads them.  Host tensors and None are skipped."""
    cur = torch.cuda.current_stream(device)
    waited = False
    for t in tensors:
        if isinstance(t, torch.Tensor) and t.is_cuda:
            if not waited and cur != stream:
                stream.wait_stream(cur)
                waited = True
            t.record_stream(stream)


def frame_buffer(cache, dtype, B, device):
    """The persistent device frame buffer [B,512,512,3] of ``cache`` for (dtype, B): a stable pointer keeps the conv
    graph's CUDA-graph cache at one entry."""
    key = (dtype, B)
    if key not in cache:
        cache[key] = torch.empty((B, 512, 512, 3), dtype=dtype, device=device)
    return cache[key]


def frame_offsets(offsets, pad_table, B):
    """The geometry argument of the models' run_post for B frames.  Per-frame offsets [B,6] (numpy array or tensor) are
    copied into the device ``pad_table`` on the current stream and its first B rows returned; one pad info
    [top,bottom,left,right,h,w] for every frame is returned as it is, None as the pad info of a 512x512 frame."""
    if offsets is None:
        return FULL_FRAME
    if np.ndim(offsets) != 2:
        return offsets
    assert tuple(np.shape(offsets)) == (B, 6), "per-frame offsets must be [B,6]"
    return pad_table[:B].copy_(torch.as_tensor(np.asarray(offsets, np.float32) if not isinstance(offsets, torch.Tensor)
                                               else offsets.float()))


class RawStager:
    """Raw host images on their way to the device: one pinned host buffer and one device buffer of the same size, grown
    on demand to at least MIN_BYTES.  Device images are not staged: the preprocessing reads them in place."""

    MIN_BYTES = 1 << 24

    def __init__(self, device):
        self.device = device
        self.host = self.dev = None

    def stage(self, images, replace_after=None, reuse_after=None):
        """Copy the host images among ``images`` (from image_tensor) into the pinned buffer; returns staging_layout's
        (offsets, total).  Before the buffers are replaced by larger ones, ``replace_after`` (the device buffer's last
        reader) is synchronized; before the pinned buffer is overwritten, ``reuse_after`` (its last H2D copy).  Each is
        an event, a stream, or None when no such work can be pending."""
        offs, total = staging_layout(images)
        if total:
            grow = self.host is None or self.host.numel() < total
            wait = replace_after if grow else reuse_after
            if wait is not None:
                wait.synchronize()
            if grow:
                n = max(total, self.MIN_BYTES)
                self.host = torch.empty(n, dtype=torch.uint8).pin_memory()
                self.dev = torch.empty(n, dtype=torch.uint8, device=self.device)
            stage_host_images(images, offs, self.host)
        return offs, total

    def upload(self, total):
        """The H2D copy of the first ``total`` staged bytes, enqueued on the current stream."""
        self.dev[:total].copy_(self.host[:total], non_blocking=True)
