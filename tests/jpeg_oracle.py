"""numpy restatement of the integer JPEG pipeline ``cv2.imencode('.jpg', bgr)`` / ``cv2.imdecode`` run with OpenCV's
default parameters (libjpeg-turbo, quality 95, 4:2:0, ISLOW DCT, standard Huffman tables, fancy upsampling), stage by
stage, as the reference for csrc/jpeg.cu.  Each function names the libjpeg stage it restates.

Coefficients are int32 [n_mcu, 6, 64]: MCUs in raster order, blocks Y0 Y1 Y2 Y3 Cb Cr, each in zig-zag order and
quantized, the layout the device buffers use."""
from __future__ import annotations

import numpy as np

from romp_b200.jpeg import HUFF_TABLES, ZIGZAG, geometry, header, huffman_codes, quant_tables

SCALEBITS, ONE_HALF = 16, 1 << 15
CBCR_OFFSET = 128 << SCALEBITS


def fix(x):
    return int(x * (1 << SCALEBITS) + 0.5)


def rgb_ycc(img):
    """jccolor.c rgb_ycc_convert (table form): BGR uint8 [H,W,3] -> Y, Cb, Cr int64 [H,W]."""
    b, g, r = (img[..., c].astype(np.int64) for c in range(3))
    y = (fix(0.29900) * r + fix(0.58700) * g + fix(0.11400) * b + ONE_HALF) >> SCALEBITS
    cb = (-fix(0.16874) * r - fix(0.33126) * g + fix(0.5) * b + CBCR_OFFSET + ONE_HALF - 1) >> SCALEBITS
    cr = (fix(0.5) * r - fix(0.41869) * g - fix(0.08131) * b + CBCR_OFFSET + ONE_HALF - 1) >> SCALEBITS
    return y, cb, cr


def _descale(x, n):
    return (x + (1 << (n - 1))) >> n


def _fdct_1d(d, final):
    """One pass of jfdctint.c jpeg_fdct_islow over the last axis (CONST_BITS 13, PASS1_BITS 2)."""
    c = [d[..., i] for i in range(8)]
    tmp0, tmp7, tmp1, tmp6 = c[0] + c[7], c[0] - c[7], c[1] + c[6], c[1] - c[6]
    tmp2, tmp5, tmp3, tmp4 = c[2] + c[5], c[2] - c[5], c[3] + c[4], c[3] - c[4]
    tmp10, tmp13, tmp11, tmp12 = tmp0 + tmp3, tmp0 - tmp3, tmp1 + tmp2, tmp1 - tmp2
    sh = 15 if final else 11
    out = [None] * 8
    out[0] = _descale(tmp10 + tmp11, 2) if final else (tmp10 + tmp11) << 2
    out[4] = _descale(tmp10 - tmp11, 2) if final else (tmp10 - tmp11) << 2
    z1 = (tmp12 + tmp13) * 4433
    out[2] = _descale(z1 + tmp13 * 6270, sh)
    out[6] = _descale(z1 - tmp12 * 15137, sh)
    z1, z2, z3, z4 = tmp4 + tmp7, tmp5 + tmp6, tmp4 + tmp6, tmp5 + tmp7
    z5 = (z3 + z4) * 9633
    tmp4, tmp5, tmp6, tmp7 = tmp4 * 2446, tmp5 * 16819, tmp6 * 25172, tmp7 * 12299
    z1, z2, z3, z4 = z1 * -7373, z2 * -20995, z3 * -16069 + z5, z4 * -3196 + z5
    out[7] = _descale(tmp4 + z1 + z3, sh)
    out[5] = _descale(tmp5 + z2 + z4, sh)
    out[3] = _descale(tmp6 + z2 + z3, sh)
    out[1] = _descale(tmp7 + z1 + z4, sh)
    return np.stack(out, -1)


def fdct_islow(blocks):
    """jpeg_fdct_islow on sample blocks [..., 8, 8] already centred (sample - 128): rows, then columns."""
    rows = _fdct_1d(blocks.astype(np.int64), False)
    return np.swapaxes(_fdct_1d(np.swapaxes(rows, -1, -2), True), -1, -2)


def quantize(coef, q):
    """jcdctmgr.c quantize with the ISLOW divisors 8*q: round half away from zero."""
    d = (q.reshape(8, 8) * 8).astype(np.int64)
    a = (np.abs(coef) + d // 2) // d
    return np.where(coef < 0, -a, a)


def _blocks(plane, bh, bw):
    """[bh*8, bw*8] -> [bh, bw, 8, 8]."""
    return plane.reshape(bh, 8, bw, 8).transpose(0, 2, 1, 3)


def forward(img, quality=95):
    """Frame -> quantized coefficients [n_mcu, 6, 64] (zig-zag), libjpeg's compressor up to the entropy coder:
    colour conversion, edge replication (jcprepct.c expand_bottom_edge, jcsample.c expand_right_edge), h2v2_downsample
    with the alternating 1, 2 bias, FDCT, quantization, and jccoefct.c's dummy blocks of partial MCUs (zero AC, the DC
    of the preceding block)."""
    h, w = img.shape[:2]
    mw, mh = geometry(h, w)
    qy, qc = quant_tables(quality)
    y, cb, cr = rgb_ycc(img)
    bw, bh = (w + 7) // 8, (h + 7) // 8                     # luma blocks that hold pixels
    rows, cols = np.minimum(np.arange(mh * 16), h - 1), np.minimum(np.arange(mw * 16), w - 1)
    yp = y[rows][:, cols]
    cw, ch = (w + 1) // 2, (h + 1) // 2                     # chroma samples that hold pixels
    crow = np.minimum(np.arange(mh * 8), ch - 1)
    bias = np.tile([1, 2], mw * 4)
    chroma = []
    for p in (cb, cr):
        pp = p[rows][:, cols]
        s = pp[0::2, 0::2] + pp[0::2, 1::2] + pp[1::2, 0::2] + pp[1::2, 1::2]
        chroma.append(((s + bias) >> 2)[crow])
    yq = quantize(fdct_islow(_blocks(yp, mh * 2, mw * 2) - 128), qy)          # [2mh, 2mw, 8, 8]
    yq = yq.reshape(mh * 2, mw * 2, 64)
    # jccoefct.c compress_data: right dummies take the DC of their left neighbour, a bottom dummy row that of the
    # MCU's last block above it (Y1, itself possibly a right dummy)
    if bw % 2:
        yq[:, bw] = 0
        yq[:, bw, 0] = yq[:, bw - 1, 0]
    if bh % 2:
        yq[bh] = 0
        yq[bh, :, 0] = np.repeat(yq[bh - 1, 1::2, 0], 2)
    yq = yq.reshape(mh, 2, mw, 2, 64).transpose(0, 2, 1, 3, 4).reshape(mh * mw, 4, 64)
    cq = [quantize(fdct_islow(_blocks(c, mh, mw) - 128), qc).reshape(mh * mw, 1, 64) for c in chroma]
    nat = np.concatenate([yq] + cq, 1)
    return nat[:, :, ZIGZAG].astype(np.int32)


def _nbits(v):
    """Bit length of |v| (jchuff.c JPEG_NBITS)."""
    a = np.abs(v).astype(np.int64)
    n = np.zeros(a.shape, np.int64)
    while np.any(a >> n):
        n += (a >> n) > 0
    return n


def _magnitude_bits(v, n):
    """The n low bits jchuff.c appends after a size code: v, or v - 1 for a negative v."""
    return np.where(v < 0, v - 1, v) & ((np.int64(1) << n) - 1)


def entropy_segment(coefs):
    """jchuff.c encode_one_block over every block in MCU order (DC prediction per component, AC run/size with ZRL and
    EOB), then finish_pass's padding with 1-bits and emit_byte's 0xFF 0x00 stuffing.  Returns the bytes between SOS and
    EOI.  Vectorized: every code is an item (block, place in the block, value, length), packed in that order."""
    codes = [huffman_codes(t) for t in HUFF_TABLES]             # DC0, AC0, DC1, AC1
    flat = coefs.reshape(-1, 64).astype(np.int64)
    nb = len(flat)
    comp = np.tile([0, 0, 0, 0, 1, 2], nb // 6)
    chroma = comp > 0
    blk_ids, keys, vals, lens = [], [], [], []

    def add(b, key, v, n):
        blk_ids.append(b); keys.append(np.broadcast_to(key, b.shape)); vals.append(v); lens.append(n)

    dc = flat[:, 0]
    pred = np.zeros(nb, np.int64)
    for c in range(3):
        idx = np.nonzero(comp == c)[0]
        pred[idx[1:]] = dc[idx[:-1]]
    diff = dc - pred
    n = _nbits(diff)
    b = np.arange(nb)
    dcc = np.where(chroma, codes[2][0][n], codes[0][0][n]).astype(np.int64)
    dcl = np.where(chroma, codes[2][1][n], codes[0][1][n]).astype(np.int64)
    add(b, 0, dcc, dcl)
    add(b, 1, _magnitude_bits(diff, n), n)
    bb, kk = np.nonzero(flat[:, 1:])
    kk = kk + 1
    first = np.r_[True, bb[1:] != bb[:-1]]
    prev = np.where(first, 0, np.r_[0, kk[:-1]])
    run = kk - prev - 1
    ch = chroma[bb]
    ac_code = np.where(ch[:, None], codes[3][0][None], codes[1][0][None]).astype(np.int64)
    ac_len = np.where(ch[:, None], codes[3][1][None], codes[1][1][None]).astype(np.int64)
    zrl = run // 16
    zc, zl = ac_code[:, 0xF0], ac_len[:, 0xF0]
    zval = np.zeros_like(zc)
    for i in range(3):
        zval = np.where(zrl > i, (zval << zl) | zc, zval)
    add(bb, 4 * kk, zval, zrl * zl)
    v = flat[bb, kk]
    n = _nbits(v)
    sym = ((run % 16) << 4) + n
    r = np.arange(len(bb))
    add(bb, 4 * kk + 1, ac_code[r, sym], ac_len[r, sym])
    add(bb, 4 * kk + 2, _magnitude_bits(v, n), n)
    last = np.zeros(nb, np.int64)
    last[bb] = kk                                                   # ascending within a block: the last one wins
    eob = np.nonzero(last < 63)[0]
    add(eob, 1000, np.where(chroma[eob], codes[3][0][0], codes[1][0][0]).astype(np.int64),
        np.where(chroma[eob], codes[3][1][0], codes[1][1][0]).astype(np.int64))
    blk_ids, keys, vals, lens = (np.concatenate(x).astype(np.int64) for x in (blk_ids, keys, vals, lens))
    order = np.lexsort((keys, blk_ids))
    vals, lens = vals[order], lens[order]
    total = int(lens.sum())
    idx = np.repeat(np.arange(len(lens)), lens)
    k = np.arange(total) - np.repeat(np.cumsum(lens) - lens, lens)
    bits = ((vals[idx] >> (lens[idx] - 1 - k)) & 1).astype(np.uint8)
    bits = np.concatenate([bits, np.ones((-total) % 8, np.uint8)])
    data = np.packbits(bits)
    ff = np.nonzero(data == 0xFF)[0]
    return np.insert(data, ff + 1, 0).tobytes()


def encode(img, quality=95):
    """The whole file: header + entropy-coded segment + EOI."""
    return header(*img.shape[:2], quality) + entropy_segment(forward(img, quality)) + b"\xff\xd9"


def _idct_1d(d, final):
    """One pass of jidctint.c jpeg_idct_islow over the last axis (the zero-AC shortcuts give the same values)."""
    c = [d[..., i] for i in range(8)]
    z2, z3 = c[2], c[6]
    z1 = (z2 + z3) * 4433
    tmp2 = z1 + z3 * -15137
    tmp3 = z1 + z2 * 6270
    tmp0, tmp1 = (c[0] + c[4]) << 13, (c[0] - c[4]) << 13
    tmp10, tmp13, tmp11, tmp12 = tmp0 + tmp3, tmp0 - tmp3, tmp1 + tmp2, tmp1 - tmp2
    t0, t1, t2, t3 = c[7], c[5], c[3], c[1]
    z1, z2, z3, z4 = t0 + t3, t1 + t2, t0 + t2, t1 + t3
    z5 = (z3 + z4) * 9633
    t0, t1, t2, t3 = t0 * 2446, t1 * 16819, t2 * 25172, t3 * 12299
    z1, z2, z3, z4 = z1 * -7373, z2 * -20995, z3 * -16069 + z5, z4 * -3196 + z5
    t0, t1, t2, t3 = t0 + z1 + z3, t1 + z2 + z4, t2 + z2 + z3, t3 + z1 + z4
    sh = 18 if final else 11
    out = [tmp10 + t3, tmp11 + t2, tmp12 + t1, tmp13 + t0, tmp13 - t0, tmp12 - t1, tmp11 - t2, tmp10 - t3]
    return np.stack([_descale(o, sh) for o in out], -1)


def idct_range_limit(x):
    """IDCT_range_limit[x & RANGE_MASK] of jdmaster.c prepare_range_limit_table: x + 128 clamped to [0, 255] for x in
    [-512, 511], wrapping around with period 1024 outside."""
    v = x & 1023
    return np.where(v < 128, v + 128, np.where(v < 512, 255, np.where(v < 896, 0, v - 896)))


def idct_islow(coef_nat, q):
    """Dequantize (jddctmgr.c ISLOW multipliers = the quantization table) and jpeg_idct_islow: [..., 8, 8] natural
    order -> samples [..., 8, 8]."""
    d = coef_nat.astype(np.int64) * q.reshape(8, 8).astype(np.int64)
    cols = np.swapaxes(_idct_1d(np.swapaxes(d, -1, -2), False), -1, -2)
    return idct_range_limit(_idct_1d(cols, True))


def _plane(blocks, bh, bw):
    return blocks.reshape(bh, bw, 8, 8).transpose(0, 2, 1, 3).reshape(bh * 8, bw * 8)


def upsample_h2v2(c, h, w):
    """jdsample.c's 2x2 upsampling of a chroma plane whose first ceil(h/2) x ceil(w/2) samples hold pixels.  Returns
    [h, w].  jinit_upsampler takes h2v2_fancy_upsample only for a chroma width above 2, else h2v2_upsample (each sample
    replicated 2 x 2).  Fancy: rows beyond the first ceil(h/2) replicate the last one (jdmainct.c set_bottom_pointers),
    the row above the first is itself (set_wraparound), and columns likewise (the SIMD variants' dummy column)."""
    ch, cw = (h + 1) // 2, (w + 1) // 2
    c = c[:ch, :cw].astype(np.int64)
    if cw <= 2:
        return c[np.arange(h) // 2][:, np.arange(w) // 2]
    up = c[np.maximum(np.arange(ch) - 1, 0)]
    down = c[np.minimum(np.arange(ch) + 1, ch - 1)]
    rows = np.empty((2 * ch, cw), np.int64)
    rows[0::2] = 3 * c + up
    rows[1::2] = 3 * c + down
    left = rows[:, np.maximum(np.arange(cw) - 1, 0)]
    right = rows[:, np.minimum(np.arange(cw) + 1, cw - 1)]
    out = np.empty((2 * ch, 2 * cw), np.int64)
    out[:, 0::2] = (3 * rows + left + 8) >> 4
    out[:, 1::2] = (3 * rows + right + 7) >> 4
    return out[:h, :w]


def ycc_bgr(y, cb, cr):
    """jdcolor.c ycc_rgb_convert (table form) to BGR uint8."""
    cbx, crx = cb - 128, cr - 128
    r = y + ((fix(1.40200) * crx + ONE_HALF) >> SCALEBITS)
    g = y + ((-fix(0.34414) * cbx + ONE_HALF - fix(0.71414) * crx) >> SCALEBITS)
    b = y + ((fix(1.77200) * cbx + ONE_HALF) >> SCALEBITS)
    return np.clip(np.stack([b, g, r], -1), 0, 255).astype(np.uint8)


def decode(coefs, h, w, quality=95):
    """Quantized coefficients [n_mcu, 6, 64] (zig-zag) of an h x w frame -> the BGR frame ``cv2.imdecode`` gives."""
    mw, mh = geometry(h, w)
    qy, qc = quant_tables(quality)
    nat = np.zeros_like(coefs)
    nat[:, :, ZIGZAG] = coefs
    nat = nat.reshape(mh, mw, 6, 8, 8)
    yb = idct_islow(nat[:, :, :4], qy).reshape(mh, mw, 2, 2, 8, 8).transpose(0, 2, 1, 3, 4, 5).reshape(mh * 2, mw * 2, 8, 8)
    y = _plane(yb, mh * 2, mw * 2)[:h, :w]
    cb = upsample_h2v2(_plane(idct_islow(nat[:, :, 4], qc), mh, mw), h, w)
    cr = upsample_h2v2(_plane(idct_islow(nat[:, :, 5], qc), mh, mw), h, w)
    return ycc_bgr(y, cb, cr)
