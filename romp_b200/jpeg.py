"""GPU JPEG round trip of the frames the command lines extract from a video (``cli.frame_source``): the bytes
``cv2.imencode('.jpg', frame)`` writes and the pixels ``cv2.imdecode`` gives back for them, with OpenCV's default
parameters (libjpeg-turbo baseline: quality 95, 4:2:0, ISLOW DCT, the standard Huffman tables, no restart markers).

The header depends only on the frame size and is composed here from the JPEG standard's Annex K tables
(ITU-T T.81); the entropy-coded segment and the decoded frame come from two CUDA entry points
(``b200romp_jpeg_encode_batch``, ``b200romp_jpeg_decode_coefs_batch``, csrc/jpeg.cu).  The decoded frame is computed
from the quantized coefficients the encoder left on the device: nothing is Huffman-decoded.
"""
from __future__ import annotations

import ctypes as C
import struct

import numpy as np

QUALITY = 95

# Annex K.1 / K.2 quantization tables, natural (row-major) order
STD_LUMA_Q = np.array([
    16, 11, 10, 16, 24, 40, 51, 61, 12, 12, 14, 19, 26, 58, 60, 55,
    14, 13, 16, 24, 40, 57, 69, 56, 14, 17, 22, 29, 51, 87, 80, 62,
    18, 22, 37, 56, 68, 109, 103, 77, 24, 35, 55, 64, 81, 104, 113, 92,
    49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100, 103, 99], np.int32)
STD_CHROMA_Q = np.full(64, 99, np.int32)
STD_CHROMA_Q[[0, 1, 2, 3, 8, 9, 10, 11, 16, 17, 18, 24, 25, 26]] = [17, 18, 24, 47, 18, 21, 26, 66, 24, 26, 56, 47, 66, 99]
# zig-zag position k -> natural index
ZIGZAG = np.array([
    0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14, 21,
    28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61,
    54, 47, 55, 62, 63], np.int32)

# Annex K.3 Huffman tables: (code counts per length 1..16, symbols)
DC_LUMA = ([0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0], list(range(12)))
DC_CHROMA = ([0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0], list(range(12)))
AC_LUMA = ([0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 0x7d], [
    0x01, 0x02, 0x03, 0x00, 0x04, 0x11, 0x05, 0x12, 0x21, 0x31, 0x41, 0x06, 0x13, 0x51, 0x61, 0x07,
    0x22, 0x71, 0x14, 0x32, 0x81, 0x91, 0xa1, 0x08, 0x23, 0x42, 0xb1, 0xc1, 0x15, 0x52, 0xd1, 0xf0,
    0x24, 0x33, 0x62, 0x72, 0x82, 0x09, 0x0a, 0x16, 0x17, 0x18, 0x19, 0x1a, 0x25, 0x26, 0x27, 0x28,
    0x29, 0x2a, 0x34, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a, 0x43, 0x44, 0x45, 0x46, 0x47, 0x48, 0x49,
    0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68, 0x69,
    0x6a, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88, 0x89,
    0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7,
    0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3, 0xc4, 0xc5,
    0xc6, 0xc7, 0xc8, 0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe1, 0xe2,
    0xe3, 0xe4, 0xe5, 0xe6, 0xe7, 0xe8, 0xe9, 0xea, 0xf1, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8,
    0xf9, 0xfa])
AC_CHROMA = ([0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 0x77], [
    0x00, 0x01, 0x02, 0x03, 0x11, 0x04, 0x05, 0x21, 0x31, 0x06, 0x12, 0x41, 0x51, 0x07, 0x61, 0x71,
    0x13, 0x22, 0x32, 0x81, 0x08, 0x14, 0x42, 0x91, 0xa1, 0xb1, 0xc1, 0x09, 0x23, 0x33, 0x52, 0xf0,
    0x15, 0x62, 0x72, 0xd1, 0x0a, 0x16, 0x24, 0x34, 0xe1, 0x25, 0xf1, 0x17, 0x18, 0x19, 0x1a, 0x26,
    0x27, 0x28, 0x29, 0x2a, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a, 0x43, 0x44, 0x45, 0x46, 0x47, 0x48,
    0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68,
    0x69, 0x6a, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x82, 0x83, 0x84, 0x85, 0x86, 0x87,
    0x88, 0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9a, 0xa2, 0xa3, 0xa4, 0xa5,
    0xa6, 0xa7, 0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3,
    0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda,
    0xe2, 0xe3, 0xe4, 0xe5, 0xe6, 0xe7, 0xe8, 0xe9, 0xea, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8,
    0xf9, 0xfa])
HUFF_TABLES = (DC_LUMA, AC_LUMA, DC_CHROMA, AC_CHROMA)


def quant_tables(quality=QUALITY):
    """(luma, chroma) quantization tables in natural order, scaled as libjpeg's jpeg_set_quality does
    (jcparam.c: jpeg_quality_scaling, then jpeg_add_quant_table with force_baseline)."""
    q = min(max(int(quality), 1), 100)
    scale = 5000 // q if q < 50 else 200 - 2 * q
    return tuple(np.clip((t * scale + 50) // 100, 1, 255).astype(np.int32) for t in (STD_LUMA_Q, STD_CHROMA_Q))


def huffman_codes(table):
    """Code and length of every symbol of a (counts, symbols) table (Annex C, as jchuff.c jpeg_make_c_derived_tbl):
    arrays indexed by symbol, length 0 for a symbol the table lacks."""
    counts, symbols = table
    code, length = np.zeros(256, np.uint32), np.zeros(256, np.int32)
    c, k = 0, 0
    for bits in range(1, 17):
        for _ in range(counts[bits - 1]):
            code[symbols[k]], length[symbols[k]] = c, bits
            c += 1
            k += 1
        c <<= 1
    return code, length


def header(h, w, quality=QUALITY):
    """The bytes of ``cv2.imencode('.jpg')`` before the entropy-coded segment for an h x w BGR frame: SOI, JFIF APP0,
    one DQT per table (zig-zag order), SOF0 (Y 2x2, Cb and Cr 1x1), the four DHTs in the order libjpeg emits them
    (DC0, AC0, DC1, AC1) and SOS.  623 bytes whatever the size."""
    assert 0 < h < 65536 and 0 < w < 65536, "a baseline JPEG is at most 65535 x 65535"
    out = bytearray(b"\xff\xd8")
    out += b"\xff\xe0" + struct.pack(">H5sBBBHHBB", 16, b"JFIF", 1, 1, 0, 1, 1, 0, 0)
    for i, t in enumerate(quant_tables(quality)):
        out += b"\xff\xdb" + struct.pack(">HB", 67, i) + bytes(t[ZIGZAG].astype(np.uint8))
    out += b"\xff\xc0" + struct.pack(">HBHHB", 17, 8, h, w, 3) + bytes([1, 0x22, 0, 2, 0x11, 1, 3, 0x11, 1])
    for cls_id, (counts, symbols) in zip((0x00, 0x10, 0x01, 0x11), HUFF_TABLES):
        out += b"\xff\xc4" + struct.pack(">HB", 3 + 16 + len(symbols), cls_id) + bytes(counts) + bytes(symbols)
    out += b"\xff\xda" + struct.pack(">HB", 12, 3) + bytes([1, 0x00, 2, 0x11, 3, 0x11, 0, 63, 0])
    return bytes(out)


def geometry(h, w):
    """(MCU columns, MCU rows) of an h x w 4:2:0 frame: 16 x 16 pixels per MCU, six blocks each (Y0 Y1 Y2 Y3 Cb Cr)."""
    return (w + 15) // 16, (h + 15) // 16


def frame_sizes(h, w):
    """Device bytes of one h x w frame in the codec's buffers (the layout include/b200romp.h documents):
    ``coefs`` int16 [6 * MCUs, 64]; ``segment``, the worst case of the stuffed entropy-coded segment: 2 * raw_cap, where
    raw_cap = 4 * ceil((1665 * blocks + 7) / 32) holds the packed bits of blocks that each take the longest codes (an
    11-bit DC size code and 11 bits, then 63 AC codes of 16 + 10 bits) and every packed byte may gain a stuffed 0x00;
    ``enc_work`` (bit offsets, packed words, an 0xFF offset per 64 packed bytes); ``dec_work`` (the Y, Cb and Cr
    planes); ``frame``, the decoded BGR frame."""
    mw, mh = geometry(h, w)
    blocks = 6 * mw * mh
    raw_cap = 4 * ((1665 * blocks + 7 + 31) // 32)
    return {"coefs": 128 * blocks, "segment": 2 * raw_cap,
            "enc_work": 16 + 16 * ((blocks + 3) // 4) + raw_cap + 4 * ((raw_cap + 63) // 64), "dec_work": 384 * mw * mh, "frame": 3 * h * w}


def _probe_image():
    """A fixed 37 x 53 frame with every feature the codec has to get right: smooth gradients, saturated colours, a
    one-pixel checkerboard and noise, and partial MCUs on both edges."""
    rng = np.random.default_rng(20261018)
    y, x = np.mgrid[0:37, 0:53]
    img = np.stack([(x * 5) % 256, (y * 7) % 256, ((x + y) % 2) * 255], -1).astype(np.uint8)
    img[20:, :26] = rng.integers(0, 256, (17, 26, 3), dtype=np.uint8)
    img[:10, 40:] = (0, 0, 255)
    return img


class FrameCodec:
    """The GPU JPEG round trip of BGR frames on one CUDA device: for each frame the bytes ``cv2.imencode('.jpg')``
    writes and the frame ``cv2.imdecode`` gives for them, as a device tensor and a host copy.

    Host frames are staged through one pinned buffer (``staging.RawStager``), the decoded frames come back through
    another, and the device buffers of a list are grown on demand to the sizes of ``frame_sizes``; all are reused by the
    next list.  The decoded device frames and their host copies are new for every list.  ``run`` may be called from several threads; the
    lists run one at a time on the codec's own stream.  Building the codec encodes and decodes a probe frame both here
    and with the installed OpenCV: when they differ, ``usable`` is False and ``reason`` says how."""

    def __init__(self, device, quality=QUALITY):
        import threading

        import torch

        from . import _lib
        from .staging import RawStager
        self.lib = _lib.load()
        self.device = torch.device(device)
        self.stream = torch.cuda.Stream(self.device)
        self.quality = quality
        self._q = np.ascontiguousarray(np.stack(quant_tables(quality)).astype(np.uint8))
        self._counts = np.zeros((4, 16), np.uint8)
        self._symbols = np.zeros((4, 256), np.uint8)
        for i, (counts, symbols) in enumerate(HUFF_TABLES):
            self._counts[i], self._symbols[i, :len(symbols)] = counts, symbols
        self._headers = {}
        self._stager = RawStager(self.device)
        self._dev = self._host = self._seg_host = None
        self._lock = threading.Lock()
        self.usable, self.reason = self._probe()

    def header(self, h, w):
        if (h, w) not in self._headers:
            self._headers[(h, w)] = header(h, w, self.quality)
        return self._headers[(h, w)]

    def _probe(self):
        import cv2
        img = _probe_image()
        try:
            [(data, _, host)], _ = self.run([img])
        except Exception as e:                          # noqa: BLE001 - reported as the reason
            return False, f"the GPU codec failed on the probe frame: {type(e).__name__}: {e}"
        ok, ref = cv2.imencode(".jpg", img)
        if not ok:
            return False, "cv2.imencode('.jpg') failed on the probe frame"
        ref = ref.tobytes()
        if data != ref:
            return False, (f"the installed OpenCV's JPEG encoder writes other bytes than the GPU codec "
                           f"({len(ref)} against {len(data)} bytes for the probe frame)")
        if not np.array_equal(host, cv2.imdecode(np.frombuffer(ref, np.uint8), cv2.IMREAD_COLOR)):
            return False, "the installed OpenCV's JPEG decoder gives other pixels than the GPU codec"
        return True, None

    def _buffer(self, nbytes):
        import torch
        if self._dev is None or self._dev.numel() < nbytes:
            self._dev = None
            self._dev = torch.empty(max(nbytes, 1 << 24), dtype=torch.uint8, device=self.device)
        return self._dev

    def run(self, frames):
        """JPEG-encode and decode a list of HxWx3 uint8 BGR frames (numpy arrays or tensors, host or device; a device
        frame is read in place when its rows are packed pixels).  Returns ([(JPEG bytes, decoded frame as a device
        tensor [h,w,3], the same as a numpy array)], event): the decoded device frames are complete at ``event``, which a
        consumer's stream waits on.  Device frames are read on the codec's stream after the work the caller's current
        stream has enqueued so far.  One host sync per list reads the byte counts and the decoded frames; the segments
        then come back through a pinned buffer in one more."""
        import torch

        from . import _lib
        from .staging import image_tensor
        images = [image_tensor(f) for f in frames]
        n = len(images)
        shapes = [(int(t.shape[0]), int(t.shape[1])) for t in images]
        sizes = [frame_sizes(h, w) for h, w in shapes]

        def offsets(key, align=256):
            offs, total = [], 0
            for s in sizes:
                offs.append(total)
                total += (s[key] + align - 1) // align * align
            return offs, total

        caller = torch.cuda.current_stream(self.device)   # the stream that produced the device frames
        with self._lock, torch.cuda.device(self.device), torch.cuda.stream(self.stream):
            staged, staged_total = self._stager.stage(images)
            if staged_total:
                self._stager.upload(staged_total)
            coef_off, coef_total = offsets("coefs")
            seg_off, seg_total = offsets("segment")
            enc_total = sum(s["enc_work"] for s in sizes)
            dec_total = sum(s["dec_work"] for s in sizes)
            base_seg = coef_total
            base_enc = base_seg + seg_total
            base_dec = (base_enc + enc_total + 255) // 256 * 256
            base_cnt = (base_dec + dec_total + 255) // 256 * 256
            buf = self._buffer(base_cnt + 4 * n)
            p0 = buf.data_ptr()
            ptrs = [t.data_ptr() if o is None else self._stager.dev.data_ptr() + o for t, o in zip(images, staged)]
            strides = [t.stride(0) if o is None else 3 * w for t, o, (_, w) in zip(images, staged, shapes)]
            hs = (C.c_int * n)(*[h for h, _ in shapes])
            ws = (C.c_int * n)(*[w for _, w in shapes])
            coefs = (C.c_void_p * n)(*[p0 + o for o in coef_off])
            segs = (C.c_void_p * n)(*[p0 + base_seg + o for o in seg_off])
            q = self._q.ctypes.data_as(C.c_void_p)
            st = C.c_void_p(self.stream.cuda_stream)
            after = [t for t, o in zip(images, staged) if o is None]
            if after:
                self.stream.wait_stream(caller)
            _lib.check(self.lib.b200romp_jpeg_encode_batch(
                (C.c_void_p * n)(*ptrs), hs, ws, (C.c_int * n)(*strides), n, q, self._counts.ctypes.data_as(C.c_void_p),
                self._symbols.ctypes.data_as(C.c_void_p), coefs, segs, C.c_void_p(p0 + base_cnt), C.c_void_p(p0 + base_enc), st),
                "jpeg_encode_batch")
            decoded = [torch.empty((h, w, 3), dtype=torch.uint8, device=self.device) for h, w in shapes]
            _lib.check(self.lib.b200romp_jpeg_decode_coefs_batch(
                coefs, hs, ws, n, q, (C.c_void_p * n)(*[d.data_ptr() for d in decoded]), C.c_void_p(p0 + base_dec), st),
                "jpeg_decode_coefs_batch")
            for t in after:
                t.record_stream(self.stream)
            counts = buf[base_cnt:base_cnt + 4 * n].view(torch.int32).to("cpu", non_blocking=True)
            frame_total = sum(s["frame"] for s in sizes)
            if self._host is None or self._host.numel() < frame_total:
                self._host = torch.empty(max(frame_total, 1 << 24), dtype=torch.uint8, pin_memory=True)
            host, o = [], 0
            for (h, w), d in zip(shapes, decoded):
                host.append(self._host[o:o + 3 * h * w].view(h, w, 3))
                host[-1].copy_(d, non_blocking=True)
                o += 3 * h * w
            event = torch.cuda.Event()
            event.record(self.stream)
            self.stream.synchronize()
            counts = counts.tolist()
            host = [hd.numpy().copy() for hd in host]          # the pinned buffer serves the next list
            if self._seg_host is None or self._seg_host.numel() < sum(counts):
                self._seg_host = torch.empty(max(sum(counts), 1 << 24), dtype=torch.uint8, pin_memory=True)
            o, spans = 0, []
            for so, c in zip(seg_off, counts):
                self._seg_host[o:o + c].copy_(buf[base_seg + so:base_seg + so + c], non_blocking=True)
                spans.append((o, o + c))
                o += c
            self.stream.synchronize()
            seg_bytes = self._seg_host[:o].numpy().tobytes()
            segments = [seg_bytes[a:b] for a, b in spans]
        out = [(self.header(h, w) + s + b"\xff\xd9", d, hd) for (h, w), s, d, hd in zip(shapes, segments, decoded, host)]
        return out, event
