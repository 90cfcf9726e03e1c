// The JPEG round trip of the frames the command lines extract from a video (cli.frame_source): the entropy-coded
// segment cv2.imencode('.jpg', frame) writes with OpenCV's defaults (libjpeg-turbo, quality 95, 4:2:0, ISLOW DCT,
// standard Huffman tables, no restart markers) and the frame cv2.imdecode gives back for it.  The decoded frame is
// computed from the quantized coefficients the encoder leaves on the device: nothing is Huffman-decoded.
//
// Encoder, per batch of frames of mixed sizes (grid z = frame):
//   jpeg_forward_kernel      one CTA per MCU: jccolor.c rgb_ycc_convert, edge replication (jcprepct.c / jcsample.c),
//                            jcsample.c h2v2_downsample (bias 1, 2, 1, 2 ...), jfdctint.c jpeg_fdct_islow, jcdctmgr.c
//                            quantize (divisor 8q, round half away from zero), jccoefct.c dummy blocks; zig-zag order
//   jpeg_block_bits_kernel   one thread per block: the bit length of jchuff.c encode_one_block's codes for the block
//   jpeg_scan_kernel         one CTA per frame: exclusive prefix sum of the bit lengths -> each block's bit offset
//   jpeg_pack_kernel         one thread per block: writes its codes at its bit offset (finish_pass's 1-bit padding
//                            after the last block)
//   jpeg_ff_count_kernel     one thread per 64 packed bytes: how many are 0xFF
//   jpeg_scan_kernel         prefix sum of those counts
//   jpeg_stuff_kernel        one thread per 64 packed bytes: scatter with a 0x00 after every 0xFF (emit_byte)
// Decoder:
//   jpeg_idct_kernel         one CTA per MCU: dequantize, jidctint.c jpeg_idct_islow with the IDCT range-limit table
//   jpeg_color_kernel        one thread per pixel: jdsample.c h2v2 (fancy) upsampling, jdcolor.c ycc_rgb_convert to BGR
// The integer rules are restated stage by stage in tests/jpeg_oracle.py and checked there against cv2.
#include <algorithm>
#include <cstring>

#include "common.cuh"

namespace b200romp {

constexpr int kJpegBatch = 16;            // frames per launch: the descriptors and tables stay inside 4 KB of parameters
constexpr int kJpegBlockBits = B200ROMP_JPEG_BLOCK_BITS;
constexpr int kJpegFFChunk = 64;          // packed bytes per 0xFF count: the stuffing pass's unit

__constant__ unsigned char c_zigzag[64] = {
    0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14, 21,
    28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61,
    54, 47, 55, 62, 63};

struct JpegGeom {
  int h, w, mw, mh;                       // pixels; MCUs (16 x 16 pixels, blocks Y0 Y1 Y2 Y3 Cb Cr)
  __host__ __device__ int mcus() const { return mw * mh; }
  __host__ __device__ int blocks() const { return 6 * mw * mh; }
};

static JpegGeom jpeg_geom(int h, int w) { return JpegGeom{h, w, (w + 15) / 16, (h + 15) / 16}; }
static size_t raw_cap_bytes(const JpegGeom& g) { return 4 * (((size_t)kJpegBlockBits * g.blocks() + 7 + 31) / 32); }
static size_t align16(size_t b) { return (b + 15) / 16 * 16; }
static size_t ff_cap_bytes(const JpegGeom& g) { return 4 * ((raw_cap_bytes(g) + kJpegFFChunk - 1) / kJpegFFChunk); }
static size_t enc_work_bytes(const JpegGeom& g) { return 16 + align16(4 * (size_t)g.blocks()) + raw_cap_bytes(g) + ff_cap_bytes(g); }

struct EncFrame {
  const unsigned char* img;
  short* coefs;                           // [blocks][64] zig-zag
  unsigned char* out;                     // entropy-coded segment, stuffed
  int* out_bytes;                         // device: its length
  unsigned* bitoff;                       // [blocks] bit lengths, then offsets
  unsigned* raw;                          // packed words before stuffing
  unsigned* ffc;                          // [packed bytes / 64] 0xFF counts, then offsets
  unsigned* totals;                       // [0] bits, [1] 0xFF bytes
  JpegGeom g;
  int row_stride;
};

struct HuffTabs {                         // jchuff.c c_derived_tbl: DC0, DC1 (sizes 0..15), AC0, AC1 (symbols 0..255)
  unsigned short dc_code[2][16];
  unsigned char dc_len[2][16];
  unsigned short ac_code[2][256];
  unsigned char ac_len[2][256];
};

struct EncBatch {
  EncFrame f[kJpegBatch];
  unsigned char q[2][64];                 // natural order
  HuffTabs t;
};
static_assert(sizeof(EncBatch) <= 4000, "encoder parameters exceed the 4 KB launch parameter space");

// ---- forward: pixels -> quantized coefficients --------------------------------------------------------------------
__device__ __forceinline__ void fdct_1d(int* d, int stride, bool final) {
  const int d0 = d[0], d1 = d[stride], d2 = d[2 * stride], d3 = d[3 * stride];
  const int d4 = d[4 * stride], d5 = d[5 * stride], d6 = d[6 * stride], d7 = d[7 * stride];
  int tmp0 = d0 + d7, tmp7 = d0 - d7, tmp1 = d1 + d6, tmp6 = d1 - d6;
  int tmp2 = d2 + d5, tmp5 = d2 - d5, tmp3 = d3 + d4, tmp4 = d3 - d4;
  const int tmp10 = tmp0 + tmp3, tmp13 = tmp0 - tmp3, tmp11 = tmp1 + tmp2, tmp12 = tmp1 - tmp2;
  const int sh = final ? 15 : 11, rnd = 1 << (sh - 1);
  d[0] = final ? (tmp10 + tmp11 + 2) >> 2 : (tmp10 + tmp11) * 4;
  d[4 * stride] = final ? (tmp10 - tmp11 + 2) >> 2 : (tmp10 - tmp11) * 4;
  int z1 = (tmp12 + tmp13) * 4433;
  d[2 * stride] = (z1 + tmp13 * 6270 + rnd) >> sh;
  d[6 * stride] = (z1 - tmp12 * 15137 + rnd) >> sh;
  z1 = tmp4 + tmp7;
  int z2 = tmp5 + tmp6, z3 = tmp4 + tmp6, z4 = tmp5 + tmp7;
  const int z5 = (z3 + z4) * 9633;
  tmp4 *= 2446; tmp5 *= 16819; tmp6 *= 25172; tmp7 *= 12299;
  z1 *= -7373; z2 *= -20995; z3 = z3 * -16069 + z5; z4 = z4 * -3196 + z5;
  d[7 * stride] = (tmp4 + z1 + z3 + rnd) >> sh;
  d[5 * stride] = (tmp5 + z2 + z4 + rnd) >> sh;
  d[3 * stride] = (tmp6 + z2 + z3 + rnd) >> sh;
  d[stride] = (tmp7 + z1 + z4 + rnd) >> sh;
}

__global__ void __launch_bounds__(256) jpeg_forward_kernel(const __grid_constant__ EncBatch b) {
  const EncFrame& f = b.f[blockIdx.z];
  const int m = blockIdx.x;
  if (m >= f.g.mcus()) return;
  const int mx = m % f.g.mw, my = m / f.g.mw, h = f.g.h, w = f.g.w;
  __shared__ int cbcr[2][16][16];
  __shared__ int blk[6][64];
  const int t = threadIdx.x, py = t >> 4, px = t & 15;
  {
    const int gy = min(my * 16 + py, h - 1), gx = min(mx * 16 + px, w - 1);   // replicate the right and bottom edges
    const unsigned char* p = f.img + (size_t)gy * f.row_stride + (size_t)gx * 3;
    const int B = p[0], G = p[1], R = p[2];
    // FIX(0.29900) = 19595, FIX(0.58700) = 38470, FIX(0.11400) = 7471, FIX(0.16874) = 11059, FIX(0.33126) = 21709,
    // FIX(0.5) = 32768, FIX(0.41869) = 27439, FIX(0.08131) = 5329; ONE_HALF = 1 << 15, CBCR_OFFSET = 128 << 16
    const int Y = (19595 * R + 38470 * G + 7471 * B + 32768) >> 16;
    cbcr[0][py][px] = (-11059 * R - 21709 * G + 32768 * B + (128 << 16) + 32767) >> 16;
    cbcr[1][py][px] = (32768 * R - 27439 * G - 5329 * B + (128 << 16) + 32767) >> 16;
    blk[(py >> 3) * 2 + (px >> 3)][(py & 7) * 8 + (px & 7)] = Y - 128;
  }
  __syncthreads();
  if (t < 128) {                          // h2v2_downsample; chroma rows beyond ceil(h/2) repeat the last one
    const int c = t >> 6, cy = (t >> 3) & 7, cx = t & 7;
    const int ey = min(my * 8 + cy, (h + 1) / 2 - 1) - my * 8;
    const int s = cbcr[c][2 * ey][2 * cx] + cbcr[c][2 * ey][2 * cx + 1] + cbcr[c][2 * ey + 1][2 * cx] + cbcr[c][2 * ey + 1][2 * cx + 1];
    blk[4 + c][cy * 8 + cx] = ((s + 1 + (cx & 1)) >> 2) - 128;
  }
  __syncthreads();
  if (t < 48) fdct_1d(&blk[t >> 3][(t & 7) * 8], 1, false);     // rows
  __syncthreads();
  if (t < 48) fdct_1d(&blk[t >> 3][t & 7], 8, true);            // columns
  __syncthreads();
  // jccoefct.c compress_data: in the last MCU column (odd luma block columns) Y1 / Y3 are dummies with the DC of their
  // left neighbour; in the last MCU row (odd luma block rows) Y2 and Y3 are dummies with the DC of Y1
  const bool rd = mx == f.g.mw - 1 && (((w + 7) >> 3) & 1), bd = my == f.g.mh - 1 && (((h + 7) >> 3) & 1);
  short* out = f.coefs + (size_t)m * 6 * 64;
  for (int i = t; i < 6 * 64; i += 256) {
    const int bi = i >> 6, k = i & 63;
    int src = bi;
    bool dummy = false;
    if (bd && (bi == 2 || bi == 3)) { src = rd ? 0 : 1; dummy = true; }
    else if (rd && (bi & 1) && bi < 4) { src = bi - 1; dummy = true; }
    int v = 0;
    if (!dummy || k == 0) {
      const int nat = c_zigzag[k];
      const int c = blk[src][nat], d = 8 * b.q[bi >= 4][nat];
      const int a = ((c < 0 ? -c : c) + (d >> 1)) / d;
      v = c < 0 ? -a : a;
    }
    out[i] = (short)v;
  }
}

// ---- entropy coding -----------------------------------------------------------------------------------------------
__device__ __forceinline__ int nbits(int v) { return 32 - __clz(v < 0 ? -v : v); }
__device__ __forceinline__ unsigned magnitude(int v, int n) { return (unsigned)(v < 0 ? v - 1 : v) & ((1u << n) - 1); }

struct BitCounter {
  unsigned bits = 0;
  __device__ void put(unsigned, int n) { bits += n; }
};

// Appends codes at a bit offset of the packed stream (MSB first).  Whole 32-bit words of the block's range are stored;
// the first and last words, shared with the neighbouring blocks, are OR-ed into the zeroed stream.
struct BitPacker {
  unsigned* raw;
  unsigned long long buf;
  int cnt;
  unsigned word;
  bool shared;
  __device__ BitPacker(unsigned* r, unsigned start) : raw(r), buf(0), cnt(start & 31), word(start >> 5), shared((start & 31) != 0) {}
  __device__ void store(unsigned v, bool atomic) {
    v = __byte_perm(v, 0, 0x0123);        // big-endian bytes
    if (atomic) atomicOr(raw + word, v);
    else raw[word] = v;
  }
  __device__ void put(unsigned v, int n) {
    buf = (buf << n) | v;
    cnt += n;
    if (cnt >= 32) {
      cnt -= 32;
      store((unsigned)(buf >> cnt), shared);
      shared = false;
      buf &= (1ull << cnt) - 1;
      ++word;
    }
  }
  __device__ void finish() {
    if (cnt > 0) store((unsigned)(buf << (32 - cnt)), true);
  }
};

// jchuff.c encode_one_block: DC difference, AC run/size with ZRL, EOB
template <class Emit>
__device__ __forceinline__ void code_block(const short* __restrict__ zz, int pred, int chroma, const HuffTabs& t, Emit& e) {
  const int diff = zz[0] - pred, n = nbits(diff);
  e.put(t.dc_code[chroma][n], t.dc_len[chroma][n]);
  if (n) e.put(magnitude(diff, n), n);
  const unsigned short* code = t.ac_code[chroma];
  const unsigned char* len = t.ac_len[chroma];
  int r = 0;
  for (int k = 1; k < 64; ++k) {
    const int v = __ldg(zz + k);
    if (v == 0) { ++r; continue; }
    for (; r > 15; r -= 16) e.put(code[0xF0], len[0xF0]);
    const int nb = nbits(v), sym = (r << 4) + nb;
    e.put(((unsigned)code[sym] << nb) | magnitude(v, nb), len[sym] + nb);
    r = 0;
  }
  if (r > 0) e.put(code[0], len[0]);
}

// the DC predictor of block i: the previous block of the same component in MCU order (Y0 Y1 Y2 Y3 Cb Cr), 0 first
__device__ __forceinline__ int dc_pred(const short* coefs, int i) {
  const int sub = i % 6;
  const int prev = sub == 0 ? i - 3 : (sub < 4 ? i - 1 : i - 6);
  return prev < 0 ? 0 : coefs[(size_t)prev * 64];
}

__global__ void __launch_bounds__(256) jpeg_block_bits_kernel(const __grid_constant__ EncBatch b) {
  const EncFrame& f = b.f[blockIdx.z];
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= f.g.blocks()) return;
  BitCounter e;
  code_block(f.coefs + (size_t)i * 64, dc_pred(f.coefs, i), i % 6 >= 4, b.t, e);
  f.bitoff[i] = e.bits;
}

__global__ void __launch_bounds__(256) jpeg_pack_kernel(const __grid_constant__ EncBatch b) {
  const EncFrame& f = b.f[blockIdx.z];
  const int i = blockIdx.x * blockDim.x + threadIdx.x, nb = f.g.blocks();
  if (i >= nb) return;
  BitPacker e(f.raw, f.bitoff[i]);
  code_block(f.coefs + (size_t)i * 64, dc_pred(f.coefs, i), i % 6 >= 4, b.t, e);
  if (i == nb - 1) {                      // finish_pass: pad the last byte with 1-bits
    const int pad = (8 - (int)(f.totals[0] & 7)) & 7;
    if (pad) e.put((1u << pad) - 1, pad);
  }
  e.finish();
}

// exclusive prefix sum over the 1024 threads of a CTA; returns the thread's offset, *total = the sum of all
__device__ __forceinline__ unsigned block_exclusive_scan(unsigned v, unsigned* total) {
  __shared__ unsigned warp_sums[32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  unsigned x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) warp_sums[warp] = x;
  __syncthreads();
  if (warp == 0) {
    unsigned s = warp_sums[lane];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const unsigned y = __shfl_up_sync(0xffffffffu, s, o);
      if (lane >= o) s += y;
    }
    warp_sums[lane] = s;
  }
  __syncthreads();
  const unsigned before = (warp ? warp_sums[warp - 1] : 0) + x - v;
  *total = warp_sums[31];
  __syncthreads();                        // warp_sums is reused by the next call
  return before;
}

__device__ __forceinline__ unsigned raw_bytes_of(const EncFrame& f) { return (f.totals[0] + 7) >> 3; }
__device__ __forceinline__ unsigned ff_chunks_of(const EncFrame& f) {
  return (raw_bytes_of(f) + kJpegFFChunk - 1) / kJpegFFChunk;
}

// stage 0: bit lengths -> bit offsets, totals[0] = bits, and the packed words zeroed; stage 1: 0xFF counts -> offsets,
// totals[1] and *out_bytes = packed bytes + 0xFF bytes
__global__ void __launch_bounds__(1024) jpeg_scan_kernel(const __grid_constant__ EncBatch b, int stage) {
  const EncFrame& f = b.f[blockIdx.x];
  unsigned* a = stage == 0 ? f.bitoff : f.ffc;
  const unsigned n = stage == 0 ? (unsigned)f.g.blocks() : ff_chunks_of(f);
  unsigned carry = 0;
  for (unsigned base = 0; base < n; base += 4 * 1024) {
    const unsigned i0 = base + 4 * threadIdx.x;
    unsigned v[4], s = 0;
#pragma unroll
    for (int j = 0; j < 4; ++j) { v[j] = i0 + j < n ? a[i0 + j] : 0; s += v[j]; }
    unsigned total;
    unsigned off = carry + block_exclusive_scan(s, &total);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if (i0 + j < n) a[i0 + j] = off;
      off += v[j];
    }
    carry += total;
  }
  if (stage == 0) {
    if (threadIdx.x == 0) f.totals[0] = carry;
    const unsigned words = (carry + 31) >> 5;
    for (unsigned i = threadIdx.x; i < words; i += 1024) f.raw[i] = 0;
  } else if (threadIdx.x == 0) {
    f.totals[1] = carry;
    *f.out_bytes = (int)(raw_bytes_of(f) + carry);
  }
}

__global__ void __launch_bounds__(256) jpeg_ff_count_kernel(const __grid_constant__ EncBatch b) {
  const EncFrame& f = b.f[blockIdx.z];
  const unsigned bytes = raw_bytes_of(f), chunks = ff_chunks_of(f);
  for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < chunks; i += gridDim.x * blockDim.x) {
    unsigned c = 0;
#pragma unroll 4
    for (int k = 0; k < kJpegFFChunk / 4; ++k) {
      const unsigned wi = i * (kJpegFFChunk / 4) + k;
      if (4 * wi >= bytes) break;
      const unsigned v = f.raw[wi];
#pragma unroll
      for (int j = 0; j < 4; ++j) c += (4 * wi + j < bytes) && ((v >> (8 * j)) & 0xFF) == 0xFF;
    }
    f.ffc[i] = c;
  }
}

__global__ void __launch_bounds__(256) jpeg_stuff_kernel(const __grid_constant__ EncBatch b) {
  const EncFrame& f = b.f[blockIdx.z];
  const unsigned bytes = raw_bytes_of(f), chunks = ff_chunks_of(f);
  for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < chunks; i += gridDim.x * blockDim.x) {
    unsigned char* o = f.out + kJpegFFChunk * i + f.ffc[i];
    for (int k = 0; k < kJpegFFChunk / 4; ++k) {
      const unsigned wi = i * (kJpegFFChunk / 4) + k;
      if (4 * wi >= bytes) break;
      const unsigned v = f.raw[wi];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        if (4 * wi + j >= bytes) break;
        const unsigned char c = (unsigned char)(v >> (8 * j));
        *o++ = c;
        if (c == 0xFF) *o++ = 0;
      }
    }
  }
}

// ---- decoder: coefficients -> BGR ---------------------------------------------------------------------------------
struct DecFrame {
  const short* coefs;
  unsigned char* out;                     // BGR, packed rows
  unsigned char* planes;                  // Y [16mh][16mw], Cb [8mh][8mw], Cr [8mh][8mw]
  JpegGeom g;
};

struct DecBatch {
  DecFrame f[kJpegBatch];
  unsigned char q[2][64];
};

// jdmaster.c prepare_range_limit_table, as IDCT_range_limit[x & RANGE_MASK]: x + 128 clamped to [0, 255] on
// [-512, 511], wrapping around with period 1024 outside
__device__ __forceinline__ unsigned char idct_range_limit(int x) {
  const int v = x & 1023;
  return (unsigned char)(v < 128 ? v + 128 : v < 512 ? 255 : v < 896 ? 0 : v - 896);
}

// one pass of jpeg_idct_islow over 8 values at stride `stride` (the zero-AC shortcuts give the same values)
__device__ __forceinline__ void idct_1d(const int* in, int stride, int (&o)[8], int sh) {
  int z2 = in[2 * stride], z3 = in[6 * stride];
  int z1 = (z2 + z3) * 4433;
  const int tmp2 = z1 + z3 * -15137, tmp3 = z1 + z2 * 6270;
  const int tmp0 = (in[0] + in[4 * stride]) * 8192, tmp1 = (in[0] - in[4 * stride]) * 8192;
  const int tmp10 = tmp0 + tmp3, tmp13 = tmp0 - tmp3, tmp11 = tmp1 + tmp2, tmp12 = tmp1 - tmp2;
  int t0 = in[7 * stride], t1 = in[5 * stride], t2 = in[3 * stride], t3 = in[stride];
  z1 = t0 + t3; z2 = t1 + t2; z3 = t0 + t2;
  int z4 = t1 + t3;
  const int z5 = (z3 + z4) * 9633;
  t0 *= 2446; t1 *= 16819; t2 *= 25172; t3 *= 12299;
  z1 *= -7373; z2 *= -20995; z3 = z3 * -16069 + z5; z4 = z4 * -3196 + z5;
  t0 += z1 + z3; t1 += z2 + z4; t2 += z2 + z3; t3 += z1 + z4;
  const int rnd = 1 << (sh - 1);
  o[0] = (tmp10 + t3 + rnd) >> sh; o[7] = (tmp10 - t3 + rnd) >> sh;
  o[1] = (tmp11 + t2 + rnd) >> sh; o[6] = (tmp11 - t2 + rnd) >> sh;
  o[2] = (tmp12 + t1 + rnd) >> sh; o[5] = (tmp12 - t1 + rnd) >> sh;
  o[3] = (tmp13 + t0 + rnd) >> sh; o[4] = (tmp13 - t0 + rnd) >> sh;
}

__global__ void __launch_bounds__(384) jpeg_idct_kernel(const __grid_constant__ DecBatch b) {
  const DecFrame& f = b.f[blockIdx.z];
  const int m = blockIdx.x;
  if (m >= f.g.mcus()) return;
  const int mx = m % f.g.mw, my = m / f.g.mw, t = threadIdx.x;
  __shared__ int ws[6][64];
  {
    const int bi = t >> 6, k = t & 63, nat = c_zigzag[k];
    ws[bi][nat] = (int)f.coefs[(size_t)m * 384 + t] * (int)b.q[bi >= 4][nat];
  }
  __syncthreads();
  if (t < 48) {                           // pass 1: columns
    int o[8];
    int* col = &ws[t >> 3][t & 7];
    idct_1d(col, 8, o, 11);
#pragma unroll
    for (int r = 0; r < 8; ++r) col[8 * r] = o[r];
  }
  __syncthreads();
  if (t < 48) {                           // pass 2: rows, then the range limit
    const int bi = t >> 3, r = t & 7;
    int o[8];
    idct_1d(&ws[bi][8 * r], 1, o, 18);
    unsigned char* dst;
    if (bi < 4) {
      const int pitch = 16 * f.g.mw;
      dst = f.planes + (size_t)(16 * my + 8 * (bi >> 1) + r) * pitch + 16 * mx + 8 * (bi & 1);
    } else {
      const int pitch = 8 * f.g.mw;
      dst = f.planes + (size_t)256 * f.g.mcus() + (size_t)(bi - 4) * 64 * f.g.mcus() + (size_t)(8 * my + r) * pitch + 8 * mx;
    }
#pragma unroll
    for (int c = 0; c < 8; ++c) dst[c] = idct_range_limit(o[c]);
  }
}

// jdsample.c: h2v2_fancy_upsample when the chroma width ceil(w/2) exceeds 2 (triangle filter, 3/4 nearer + 1/4 farther,
// vertically then horizontally with the rounding 8 / 7 of the left / right output; edge samples repeat), else
// h2v2_upsample (each sample 2 x 2)
__device__ __forceinline__ int chroma_at(const unsigned char* c, int pitch, int ch, int cw, int y, int x) {
  const int ci = y >> 1, cj = x >> 1;
  if (cw <= 2) return c[ci * pitch + cj];
  const int far = (y & 1) ? min(ci + 1, ch - 1) : max(ci - 1, 0);
  const int nj = (x & 1) ? min(cj + 1, cw - 1) : max(cj - 1, 0);
  const int here = 3 * c[ci * pitch + cj] + c[far * pitch + cj];
  const int side = 3 * c[ci * pitch + nj] + c[far * pitch + nj];
  return (3 * here + side + ((x & 1) ? 7 : 8)) >> 4;
}

__global__ void __launch_bounds__(256) jpeg_color_kernel(const __grid_constant__ DecBatch b) {
  const DecFrame& f = b.f[blockIdx.z];
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
  if (x >= f.g.w || y >= f.g.h) return;
  const int pitch_y = 16 * f.g.mw, pitch_c = 8 * f.g.mw, ch = (f.g.h + 1) / 2, cw = (f.g.w + 1) / 2;
  const unsigned char* cb_plane = f.planes + (size_t)256 * f.g.mcus();
  const int Y = f.planes[(size_t)y * pitch_y + x];
  const int cb = chroma_at(cb_plane, pitch_c, ch, cw, y, x) - 128;
  const int cr = chroma_at(cb_plane + (size_t)64 * f.g.mcus(), pitch_c, ch, cw, y, x) - 128;
  // jdcolor.c build_ycc_rgb_table: FIX(1.40200) = 91881, FIX(1.77200) = 116130, FIX(0.71414) = 46802,
  // FIX(0.34414) = 22554
  const int R = Y + ((91881 * cr + 32768) >> 16);
  const int G = Y + ((-22554 * cb + 32768 - 46802 * cr) >> 16);
  const int B = Y + ((116130 * cb + 32768) >> 16);
  unsigned char* o = f.out + ((size_t)y * f.g.w + x) * 3;
  o[0] = (unsigned char)min(max(B, 0), 255);
  o[1] = (unsigned char)min(max(G, 0), 255);
  o[2] = (unsigned char)min(max(R, 0), 255);
}

// jchuff.c jpeg_make_c_derived_tbl from (counts per length, symbols); -1 for a table that is not a valid code
static int derive_huff(const unsigned char* counts, const unsigned char* symbols, int max_symbol, unsigned short* code,
                       unsigned char* len) {
  int k = 0;
  unsigned c = 0;
  for (int bits = 1; bits <= 16; ++bits) {
    for (int i = 0; i < counts[bits - 1]; ++i, ++k) {
      if (k >= 256 || symbols[k] > max_symbol || c >= (1u << bits)) return -1;
      code[symbols[k]] = (unsigned short)c++;
      len[symbols[k]] = (unsigned char)bits;
    }
    c <<= 1;
  }
  return 0;
}

}  // namespace b200romp

using namespace b200romp;

extern "C" int b200romp_jpeg_encode_batch(const unsigned char* const* imgs_bgr, const int* h, const int* w, const int* row_stride_bytes,
                                          int n, const unsigned char* qtables, const unsigned char* huff_counts,
                                          const unsigned char* huff_symbols, short* const* coefs, unsigned char* const* out,
                                          int* out_bytes, void* work, b200romp_stream stream) {
  B2R_REQUIRE(imgs_bgr && h && w && row_stride_bytes && n > 0 && qtables && huff_counts && huff_symbols && coefs && out &&
              out_bytes && work, "jpeg_encode_batch: bad arguments");
  for (int i = 0; i < n; ++i)
    B2R_REQUIRE(imgs_bgr[i] && coefs[i] && out[i] && h[i] > 0 && w[i] > 0 && h[i] < 65536 && w[i] < 65536 &&
                row_stride_bytes[i] >= 3 * w[i], "jpeg_encode_batch: bad frame %d", i);
  for (int i = 0; i < 128; ++i) B2R_REQUIRE(qtables[i] > 0, "jpeg_encode_batch: a quantization step is 0");
  static thread_local EncBatch batch;
  memset(&batch.t, 0, sizeof(batch.t));
  memcpy(batch.q, qtables, 128);
  for (int c = 0; c < 2; ++c) {           // huff order DC0, AC0, DC1, AC1
    B2R_REQUIRE(derive_huff(huff_counts + 16 * (2 * c), huff_symbols + 256 * (2 * c), 15, batch.t.dc_code[c], batch.t.dc_len[c]) == 0 &&
                derive_huff(huff_counts + 16 * (2 * c + 1), huff_symbols + 256 * (2 * c + 1), 255, batch.t.ac_code[c], batch.t.ac_len[c]) == 0,
                "jpeg_encode_batch: bad Huffman table %d", c);
    for (int s = 0; s <= 11; ++s) B2R_REQUIRE(batch.t.dc_len[c][s], "jpeg_encode_batch: DC table %d lacks size %d", c, s);
    for (int r = 0; r < 16; ++r)
      for (int s = 1; s <= 10; ++s) B2R_REQUIRE(batch.t.ac_len[c][(r << 4) + s], "jpeg_encode_batch: AC table %d lacks symbol %d", c, (r << 4) + s);
    B2R_REQUIRE(batch.t.ac_len[c][0] && batch.t.ac_len[c][0xF0], "jpeg_encode_batch: AC table %d lacks EOB / ZRL", c);
  }
  cudaStream_t st = (cudaStream_t)stream;
  unsigned char* wp = (unsigned char*)work;
  for (int i0 = 0; i0 < n; i0 += kJpegBatch) {
    const int nb = n - i0 < kJpegBatch ? n - i0 : kJpegBatch;
    int max_mcus = 0, max_blocks = 0;
    size_t max_chunks = 0;
    for (int j = 0; j < nb; ++j) {
      const int i = i0 + j;
      EncFrame& f = batch.f[j];
      f.g = jpeg_geom(h[i], w[i]);
      f.img = imgs_bgr[i]; f.row_stride = row_stride_bytes[i];
      f.coefs = coefs[i]; f.out = out[i]; f.out_bytes = out_bytes + i;
      const size_t cap = raw_cap_bytes(f.g);
      f.totals = (unsigned*)wp;
      f.bitoff = (unsigned*)(wp + 16);
      f.raw = (unsigned*)(wp + 16 + align16(4 * (size_t)f.g.blocks()));
      f.ffc = (unsigned*)((unsigned char*)f.raw + cap);
      wp += enc_work_bytes(f.g);
      max_mcus = max(max_mcus, f.g.mcus());
      max_blocks = max(max_blocks, f.g.blocks());
      max_chunks = std::max(max_chunks, (cap + kJpegFFChunk - 1) / kJpegFFChunk);
    }
    const int chunk_ctas = (int)std::min<size_t>((max_chunks + 255) / 256, 512);
    jpeg_forward_kernel<<<dim3(max_mcus, 1, nb), 256, 0, st>>>(batch);
    jpeg_block_bits_kernel<<<dim3((max_blocks + 255) / 256, 1, nb), 256, 0, st>>>(batch);
    jpeg_scan_kernel<<<nb, 1024, 0, st>>>(batch, 0);
    jpeg_pack_kernel<<<dim3((max_blocks + 255) / 256, 1, nb), 256, 0, st>>>(batch);
    jpeg_ff_count_kernel<<<dim3(chunk_ctas, 1, nb), 256, 0, st>>>(batch);
    jpeg_scan_kernel<<<nb, 1024, 0, st>>>(batch, 1);
    jpeg_stuff_kernel<<<dim3(chunk_ctas, 1, nb), 256, 0, st>>>(batch);
    B2R_CUDA_OK(cudaGetLastError());
  }
  return B200ROMP_OK;
}

extern "C" int b200romp_jpeg_decode_coefs_batch(const short* const* coefs, const int* h, const int* w, int n,
                                                const unsigned char* qtables, unsigned char* const* out_bgr, void* work,
                                                b200romp_stream stream) {
  B2R_REQUIRE(coefs && h && w && n > 0 && qtables && out_bgr && work, "jpeg_decode_coefs_batch: bad arguments");
  for (int i = 0; i < n; ++i)
    B2R_REQUIRE(coefs[i] && out_bgr[i] && h[i] > 0 && w[i] > 0 && h[i] < 65536 && w[i] < 65536, "jpeg_decode_coefs_batch: bad frame %d", i);
  DecBatch batch;
  memcpy(batch.q, qtables, 128);
  cudaStream_t st = (cudaStream_t)stream;
  unsigned char* wp = (unsigned char*)work;
  for (int i0 = 0; i0 < n; i0 += kJpegBatch) {
    const int nb = n - i0 < kJpegBatch ? n - i0 : kJpegBatch;
    int max_mcus = 0, max_h = 0, max_w = 0;
    for (int j = 0; j < nb; ++j) {
      const int i = i0 + j;
      DecFrame& f = batch.f[j];
      f.g = jpeg_geom(h[i], w[i]);
      f.coefs = coefs[i]; f.out = out_bgr[i]; f.planes = wp;
      wp += (size_t)384 * f.g.mcus();
      max_mcus = max(max_mcus, f.g.mcus()); max_h = max(max_h, h[i]); max_w = max(max_w, w[i]);
    }
    jpeg_idct_kernel<<<dim3(max_mcus, 1, nb), 384, 0, st>>>(batch);
    jpeg_color_kernel<<<dim3((max_w + 255) / 256, max_h, nb), 256, 0, st>>>(batch);
    B2R_CUDA_OK(cudaGetLastError());
  }
  return B200ROMP_OK;
}
