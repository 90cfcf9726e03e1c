// Fused HRNet BasicBlock on the wgmma engine: y = relu(conv2(relu(conv1(x) + b1)) + b2 + x) for 3x3 stride-1 convs of
// 64 -> 64 -> 64 channels, bf16 NHWC, one kernel per block.
//
// Unfused, a block moves five activation passes through HBM (conv1 reads x and writes t, conv2 reads t, re-reads x as its
// residual and writes y).  Here the intermediate t lives only in shared memory and the residual is taken from the staged
// input halo, so a block reads x once and writes y once.
//
// FOLD = true runs a 32-channel block on the pixel-pair view [B, H, W/2, 64] with the folded 64x64 weights of
// net.cu fold_pixel_pairs; the all-zero tap halves are skipped at compile time.
//
// Both convs run with the weights as the wgmma A operand (M = the 64 output channels, one m64) and the pixels as B (N up
// to 192), so the accumulators are channel-major: row = output channel, column = pixel.  A K-major B operand has the
// layout of a K-major A operand, so the pixels are addressed as in conv_tc.cu (8-pixel groups, taps as shifted start
// addresses) and the weight image is the one conv_tc.cu uses for B.  Per k-step an m64nNk16 reads 2 KB of weights and
// N * 32 B of pixels; with both warpgroups, conv1 + conv2 read 16 + 12 KB per k-step folded and 12 + 8 KB at 64 channels,
// against 24 + 16 KB and 16 + 8 KB when the pixels were A and every MMA was m64n64 (tools/wgmma_swap_probe.cu checks on the
// GPU that the swapped MMAs give the transposed sums bit for bit).
//
// Geometry, per 16 x TW output tile at (y0, x0) of frame n (pixel pairs when folded); TW = 8 for C = 64, 16 folded, and
// HW = TW + 4 the halo width:
//   input stage: ONE TMA load of the 20 x HW halo at (x0-2, y0-2), channels innermost, 128 B swizzle, zeros outside the
//            frame.  Halo pixel (hy, hx) is stage row hy*HW + hx.
//   conv1:   over a LINEAR domain: mid pixel (my, mx), my < 18, mx < TW + 2, is GEMM column my*HW + mx, so tap (r, s) is
//            the stage shifted by r*HW + s rows and the 8-pixel groups are contiguous (SBO = 1024 B).  Pixels up to
//            17*HW + TW + 1 are needed (213 / 357), padded to 256 / 384: warpgroup g computes the g-th half as one N = 128 /
//            N = 192 MMA per k-step.  Columns >= TW + 2 of a mid row and the padding pixels are never read by conv2; the
//            stage rows TMA never writes (from 20*HW on) feed only those.
//   mid:     relu(acc + b1) -> bf16, stored transposed (stmatrix .trans) to the mid buffer in the pixel-major swizzled
//            layout wgmma reads (16 B chunk ^ (row & 7)); then, on tiles at the frame's edge, the mid pixels outside the
//            frame are zeroed (the unfused conv2 reads TMA zero fill there).
//   conv2:   on the mid buffer: 8-pixel groups, SBO = HW rows, tap (r, s) shifted by r*HW + s rows.  Warpgroup g computes
//            one N = 128 (folded: output columns 8g..8g+7 of all 16 rows) or N = 64 (output rows 8g..8g+7) MMA per k-step.
//   output:  (acc + b2) + x, ReLU, bf16.  x at the output pixels is the interior of the halo, read in the accumulator
//            layout (ldmatrix .trans) before the stage is handed back.  Lanes l and l ^ 4 swap one value per pair of
//            channels, so each store writes 2 adjacent channels of one pixel and a warp's store 16 B of each of 8 pixels.
// Both convs keep the K order of conv_tc_kernel (taps 0..8 x 32-byte k-steps, the same folded halves skipped), so the fp32
// sums and therefore t and y are bit-identical to the unfused path.
//
// Shared memory: both convs' weights stay resident next to ONE input stage and the mid buffer.  A 64-channel conv takes
// 72 KB: with a 16x8 tile (36 KB stage, 32 KB mid) that is 212 KB of the 227 KB.  The folded weights hold only the halves
// the MMAs read: the three s = 0 taps as full 64 x 128 B tiles (128 B swizzle), the six s = -1 / s = +1 taps as 64 x 64 B
// tiles of the 32 input channels they use (64 B swizzle, w_tap_off), so a folded conv takes 48 KB.  The freed room holds a
// 16x16 tile (54 KB stage, 48 KB mid; 200 KB in all): conv1 computes 384 pixels for 256 outputs instead of 256 for 128, so
// a folded block does 15/18 of the MMA work per output pixel pair of a 16x8 tile, and the per-tile fixed costs (barriers,
// pipeline drains, the halo's two extra columns) are spread over twice the pixels.  With one stage both consumer
// warpgroups work on the same tile; the stage goes back to the producer once conv1 has retired, so the next tile's TMA
// load overlaps the mid epilogue, conv2 and the output epilogue.
// A folded variant that kept the 16x8 tile, spent the freed 48 KB on a second input stage and issued conv1 of tile j + 1
// right after conv2 of tile j (so it ran through tile j's output epilogue) measured 155.4 us per block against 154.5 us
// (H100 80GB HBM3, 700 W, batch 64 at 128^2), so it was not kept: hiding the output epilogue is not what the remaining gap
// to the operand-fetch bound is made of.
#include "conv_tc.cuh"
#include "tc_device.cuh"

namespace b200romp {

namespace {

constexpr int kBlkThreads = 384;                        // warp 0 = TMA producer, warpgroups 1, 2 = consumers
constexpr int kRowB = 128;                              // one pixel row: 64 bf16 channels = one 128 B swizzle span
constexpr int kHaloH = 20;                              // input halo of a 16-row output tile, two 3x3 convs deep
constexpr int kTapBytes = 64 * kRowB;                   // one tap of one conv: 64 output x 64 input channels
constexpr int kHalfTapBytes = 64 * 64;                  // the used half of a folded s = -1 / +1 tap: 64 x 32, 64 B rows

template <bool FOLD>
struct BlkCfg {
  static constexpr int kWBytes = FOLD ? 3 * (kTapBytes + 2 * kHalfTapBytes) : 9 * kTapBytes;   // per conv
  static constexpr int kTW = FOLD ? 16 : 8;                 // output tile width; the height is 16
  static constexpr int kHaloW = kTW + 4;
  static constexpr int kN1 = FOLD ? 192 : 128;              // conv1 mid pixels per warpgroup (wgmma N)
  static constexpr int kN2 = 8 * kTW;                       // conv2 output pixels per warpgroup (wgmma N)
  static constexpr int kG2 = kN2 / 8;                       // their 8-pixel groups, one output row each
  static constexpr int kMidRows = 2 * kN1;
  static constexpr int kStagePayload = kHaloH * kHaloW * kRowB;                                   // what TMA writes
  static constexpr int kStageBytes = ((kMidRows + 2 * kHaloW + 2) * kRowB + 1023) / 1024 * 1024;  // + what padded rows read
  static constexpr int kMidBytes = kMidRows * kRowB;
  static constexpr int kSmemBytes = 2 * kWBytes + kStageBytes + kMidBytes + 1024 /*barriers*/ + 1024 /*align slack*/;
  static_assert(17 * kHaloW + kTW + 1 < kMidRows, "conv1 blocks do not cover the mid pixels conv2 reads");
  static_assert(kHaloH * kHaloW - 2 * kHaloW - 2 > 17 * kHaloW + kTW + 1, "an unwritten stage row feeds a mid row conv2 reads");
  static_assert(kSmemBytes <= 227 * 1024, "fused block does not fit shared memory");
  static_assert(kWBytes % kTapBytes == 0, "weights are copied in tap-sized pieces");
};

// byte offset of tap `tap` in a conv's weight image.  Folded, each kernel row r holds [s = -1 half | s = 0 full | s = +1 half]
// in 16 KB, so every full tile starts 1024 B-aligned (128 B swizzle) and every half tile 512 B-aligned (64 B swizzle).
__host__ __device__ constexpr int w_tap_off(bool fold, int tap) {
  return !fold ? tap * kTapBytes
               : (tap / 3) * (kTapBytes + 2 * kHalfTapBytes) + (tap % 3 == 0 ? 0 : tap % 3 == 1 ? kHalfTapBytes : kHalfTapBytes + kTapBytes);
}

// the MMAs of a pixel-pair folded conv that only meet all-zero weights: first pixel (k-steps 0, 1) of the s = -1 taps,
// second pixel (k-steps 2, 3) of the s = +1 taps (net.cu fold_pixel_pairs, the kmask of the unfused path)
template <bool FOLD>
__device__ __forceinline__ constexpr bool blk_skip(int tap, int k) {
  return FOLD && ((tap % 3 == 0 && k < 2) || (tap % 3 == 2 && k >= 2));
}

// A descriptor of k-step k of tap `tap` (k not skipped): a half tile holds the two k-steps its tap reads
template <bool FOLD>
__device__ __forceinline__ uint64_t w_desc(uint32_t w_base, int tap, int k) {
  const uint32_t t = w_base + (uint32_t)w_tap_off(FOLD, tap);
  if (FOLD && tap % 3 != 1) return make_smem_desc(t + (k & 1) * 32, 8 * 64, kSw64);
  return make_smem_desc(t + k * 32, 8 * kRowB, kSw128);
}

// barrier over both consumer warpgroups (id 1; 0 is __syncthreads)
__device__ __forceinline__ void consumers_bar_sync() { asm volatile("bar.sync 1, 256;" ::: "memory"); }

// four 8 x 8 bf16 matrices between shared memory (rows = pixels, 16 B of channels each; lane i supplies row i % 8 of
// matrix i / 8) and the channel-major accumulator fragment (lane l: channel l / 4, pixels 2 (l % 4) + {0, 1})
__device__ __forceinline__ void ldmatrix_x4_trans(uint32_t (&r)[4], uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(addr));
}
__device__ __forceinline__ void stmatrix_x4_trans(uint32_t addr, const uint32_t (&r)[4]) {
  asm volatile("stmatrix.sync.aligned.m8n8.x4.trans.shared.b16 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(r[0]), "r"(r[1]), "r"(r[2]),
               "r"(r[3])
               : "memory");
}
__device__ __forceinline__ void st_shared_zero16(uint32_t addr) {
  asm volatile("st.shared.v4.b32 [%0], {%1, %1, %1, %1};" ::"r"(addr), "r"(0) : "memory");
}
template <int N>
__device__ __forceinline__ void wgmma_bf16(float (&d)[N / 2], uint64_t a, uint64_t b, uint32_t scale_d) {
  if constexpr (N == 192) wgmma_n192_bf16(d, a, b, scale_d);
  else if constexpr (N == 128) wgmma_n128_bf16(d, a, b, scale_d);
  else wgmma_n64(d, a, b, scale_d, false);
}
// an opaque copy: keeps the compiler from hoisting everything derived from a loop-invariant value (the ~100 shared-memory
// descriptors, the bias loads) out of the tile loop, which would pin them in registers and spill
template <typename T>
__device__ __forceinline__ T opaque(T v) {
  uint64_t u = (uint64_t)v;
  asm volatile("mov.b64 %0, %0;" : "+l"(u));
  return (T)u;
}
__device__ __forceinline__ uint32_t pack_bf16x2(float a, float b) {
  const __nv_bfloat162 v = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<const uint32_t*>(&v);
}

// one consumer thread: warpgroup g, warp w of it, lane l.  In every accumulator it holds output channels 16w + l/4 + 8e
// (e = 0, 1) of pixels 8j + 2 (l % 4) + {0, 1}: registers 4j + 2e + {0, 1}.
struct BlkThread {
  int g, w, l;
};
// conv2 of warpgroup g covers output pixels (oy0 + j, ox0 + i), j < kG2, i < 8: folded, the 8-column half g of all 16 rows;
// otherwise rows 8g .. 8g + 7.  Either way its 8-pixel groups lie kHaloW mid rows apart.
template <bool FOLD>
__device__ __forceinline__ int c2_oy0(int g) { return FOLD ? 0 : 8 * g; }
template <bool FOLD>
__device__ __forceinline__ int c2_ox0(int g) { return FOLD ? 8 * g : 0; }
struct BlkTile {
  int n, y0, x0;
  __device__ BlkTile(int tile, int tiles_x, int per_frame, int tw) {
    n = tile / per_frame;
    const int rem = tile % per_frame;
    y0 = (rem / tiles_x) * 16;
    x0 = (rem % tiles_x) * tw;
  }
};

// conv1 over the stage at a_base: mid pixels row0 .. row0 + kN1 - 1 as the B operand (8-pixel groups 1024 B apart), the
// weights as A.  Issued and committed as one group.
template <bool FOLD>
__device__ __forceinline__ void conv1_issue(float (&acc)[BlkCfg<FOLD>::kN1 / 2], uint32_t a_base, uint32_t w1_base, int row0) {
  constexpr int kHaloW = BlkCfg<FOLD>::kHaloW, kN1 = BlkCfg<FOLD>::kN1;
#pragma unroll
  for (int j = 0; j < kN1 / 2; ++j) acc[j] = 0.f;
  uint32_t scale_d = 0;
  wgmma_fence();
#pragma unroll
  for (int tap = 0; tap < 9; ++tap) {
    const uint32_t b_tap = a_base + (uint32_t)((row0 + (tap / 3) * kHaloW + tap % 3) * kRowB);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      if (blk_skip<FOLD>(tap, k)) continue;
      wgmma_bf16<kN1>(acc, w_desc<FOLD>(w1_base, tap, k), make_smem_desc(b_tap + k * 32, 8 * kRowB, kSw128), scale_d);
      scale_d = 1;
    }
  }
  wgmma_commit();
}

// residual = the block input at this thread's conv2 pixels, in the accumulator layout: output pixel (y, x) is halo pixel
// (y + 2, x + 2) of the stage at a_base.  rv[j][e] = channel 16w + l/4 + 8e of pixels 8j + 2 (l % 4) + {0, 1}.
template <bool FOLD>
__device__ __forceinline__ void load_residual(uint32_t (&rv)[BlkCfg<FOLD>::kG2][2], uint32_t a_base, const BlkThread& th) {
  constexpr int kHaloW = BlkCfg<FOLD>::kHaloW;
  const int q = th.l >> 3;   // the matrix this lane addresses: group j0 + q / 2, channel chunk 2w + q % 2
#pragma unroll
  for (int j0 = 0; j0 < BlkCfg<FOLD>::kG2; j0 += 2) {
    const int hr = (c2_oy0<FOLD>(th.g) + j0 + (q >> 1) + 2) * kHaloW + c2_ox0<FOLD>(th.g) + (th.l & 7) + 2;
    uint32_t r[4];
    ldmatrix_x4_trans(r, a_base + hr * kRowB + (((2 * th.w + (q & 1)) ^ (hr & 7)) << 4));
    rv[j0][0] = r[0]; rv[j0][1] = r[1]; rv[j0 + 1][0] = r[2]; rv[j0 + 1][1] = r[3];
  }
}

// relu(acc + b1), bf16, stored transposed to the mid buffer in the pixel-major swizzled layout wgmma reads (16 B chunk ^
// (row & 7)); then, on tiles at the frame's edge, zero the mid pixels outside the frame (the unfused conv2 reads TMA zero
// fill there).  Those lie on the ring my = 0, my = 17, mx = 0, mx = TW + 1 around the tile, so the test runs once per
// ring pixel instead of once per accumulator pixel.  Mid rows conv2 never reads (mx >= TW + 2, padding) keep any value.
template <bool FOLD>
__device__ __forceinline__ void mid_epilogue(const float (&acc)[BlkCfg<FOLD>::kN1 / 2], uint32_t mid_base, const float* b1p, const ConvParams& p,
                                             const BlkTile& tl, const BlkThread& th, int row0) {
  constexpr int kHaloW = BlkCfg<FOLD>::kHaloW, kTW = BlkCfg<FOLD>::kTW, kN1 = BlkCfg<FOLD>::kN1;
  const float bias[2] = {__ldg(b1p + 16 * th.w + (th.l >> 2)), __ldg(b1p + 16 * th.w + (th.l >> 2) + 8)};
  const int q = th.l >> 3;
#pragma unroll
  for (int j0 = 0; j0 < kN1 / 8; j0 += 2) {
    uint32_t r[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {   // matrix i: pixel group j0 + i / 2, channel e = i % 2
      const int j = j0 + (i >> 1), e = i & 1;
      r[i] = pack_bf16x2(fmaxf(acc[4 * j + 2 * e] + bias[e], 0.f), fmaxf(acc[4 * j + 2 * e + 1] + bias[e], 0.f));
    }
    const int m = row0 + 8 * (j0 + (q >> 1)) + (th.l & 7);
    stmatrix_x4_trans(mid_base + m * kRowB + (((2 * th.w + (q & 1)) ^ (m & 7)) << 4), r);
  }
  if (tl.y0 > 0 && tl.x0 > 0 && tl.y0 + 16 < p.Hout && tl.x0 + kTW < p.Wout) return;
  // each warp overwrites the two 16 B channel chunks (2w, 2w + 1) it stored, of the ring pixels in its warpgroup's rows
  __syncwarp();
  constexpr int kRingRow = kTW + 2, kRing = 2 * kRingRow + 2 * 18;
#pragma unroll 1
  for (int i = th.l; i < 2 * kRing; i += 32) {
    const int k = i >> 1;
    const int my = k < 2 * kRingRow ? (k < kRingRow ? 0 : 17) : (k - 2 * kRingRow) % 18;
    const int mx = k < 2 * kRingRow ? k % kRingRow : (k - 2 * kRingRow < 18 ? 0 : kTW + 1);
    const int m = my * kHaloW + mx;
    if (m >= row0 && m < row0 + kN1 && ((unsigned)(tl.y0 - 1 + my) >= (unsigned)p.Hout || (unsigned)(tl.x0 - 1 + mx) >= (unsigned)p.Wout))
      st_shared_zero16(mid_base + m * kRowB + (((2 * th.w + (i & 1)) ^ (m & 7)) << 4));
  }
}

// conv2 over the mid buffer: this warpgroup's kN2 output pixels (c2_oy0 / c2_ox0) as the B operand, 8-pixel groups
// kHaloW mid rows apart, the weights as A.  Issued and committed as one group.
template <bool FOLD>
__device__ __forceinline__ void conv2_issue(float (&acc2)[BlkCfg<FOLD>::kN2 / 2], uint32_t mid_base, uint32_t w2_base, int g) {
  constexpr int kHaloW = BlkCfg<FOLD>::kHaloW, kN2 = BlkCfg<FOLD>::kN2;
#pragma unroll
  for (int j = 0; j < kN2 / 2; ++j) acc2[j] = 0.f;
  uint32_t scale_d = 0;
  wgmma_fence();
#pragma unroll
  for (int tap = 0; tap < 9; ++tap) {
    const uint32_t b_tap = mid_base + (uint32_t)(((c2_oy0<FOLD>(g) + tap / 3) * kHaloW + c2_ox0<FOLD>(g) + tap % 3) * kRowB);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      if (blk_skip<FOLD>(tap, k)) continue;
      wgmma_bf16<kN2>(acc2, w_desc<FOLD>(w2_base, tap, k), make_smem_desc(b_tap + k * 32, kHaloW * kRowB, kSw128), scale_d);
      scale_d = 1;
    }
  }
  wgmma_commit();
}

// (acc + b2) + x, ReLU, bf16 (the order of the unfused conv2).  A thread holds channels c, c + 8 of pixel pairs; lanes
// l and l ^ 4 (channels c, c ^ 1) swap one value so each stores 2 adjacent channels of one pixel: a warp's store covers
// 16 B of each of 8 pixels.
template <bool FOLD>
__device__ __forceinline__ void out_epilogue(const float (&acc2)[BlkCfg<FOLD>::kN2 / 2], const uint32_t (&rv)[BlkCfg<FOLD>::kG2][2],
                                             const float* b2p, const ConvParams& p, const BlkTile& tl, const BlkThread& th) {
  __nv_bfloat16* out = reinterpret_cast<__nv_bfloat16*>(p.out);
  const int c = 16 * th.w + (th.l >> 2);
  const float bias[2] = {__ldg(b2p + c), __ldg(b2p + c + 8)};
  const int odd = (th.l >> 2) & 1;
  const int x = tl.x0 + c2_ox0<FOLD>(th.g) + 2 * (th.l & 3) + odd;   // the pixel this lane stores
#pragma unroll
  for (int j = 0; j < BlkCfg<FOLD>::kG2; ++j) {
    uint16_t h[2][2];
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const float2 r = res_pair(rv[j][e]);
      const float a = (acc2[4 * j + 2 * e] + bias[e]) + r.x, b = (acc2[4 * j + 2 * e + 1] + bias[e]) + r.y;
      h[e][0] = __bfloat16_as_ushort(__float2bfloat16_rn(fmaxf(a, 0.f)));
      h[e][1] = __bfloat16_as_ushort(__float2bfloat16_rn(fmaxf(b, 0.f)));
    }
    // even lanes keep pixel 0 and send pixel 1, odd lanes the other way round
    const uint32_t send = odd ? (uint32_t)h[0][0] | ((uint32_t)h[1][0] << 16) : (uint32_t)h[0][1] | ((uint32_t)h[1][1] << 16);
    const uint32_t recv = __shfl_xor_sync(0xffffffffu, send, 4);
    const size_t pix = ((size_t)tl.n * p.Hout + tl.y0 + c2_oy0<FOLD>(th.g) + j) * p.Wout + x;
    uint32_t* o = reinterpret_cast<uint32_t*>(out + pix * p.out_C + p.out_c_off + (c & ~1));
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const uint32_t theirs = (recv >> (16 * e)) & 0xFFFFu;
      o[4 * e] = odd ? (theirs | ((uint32_t)h[e][1] << 16)) : ((uint32_t)h[e][0] | (theirs << 16));
    }
  }
}

}  // namespace

template <bool FOLD>
__global__ void __launch_bounds__(kBlkThreads, 1)
conv_block_tc_kernel(const __grid_constant__ CUtensorMap tmap, const ConvParams p, const uint8_t* __restrict__ w1pack,
                     const uint8_t* __restrict__ w2pack, const float* __restrict__ bias1, int tiles_x, int tiles_y, int num_tiles) {
  using Cfg = BlkCfg<FOLD>;
  constexpr int kWBytes = Cfg::kWBytes, kStageBytes = Cfg::kStageBytes;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* sW1 = smem;
  uint8_t* sW2 = smem + kWBytes;
  uint8_t* sA = smem + 2 * kWBytes;
  uint8_t* sMid = sA + kStageBytes;
  uint64_t* full = reinterpret_cast<uint64_t*>(sMid + Cfg::kMidBytes);
  uint64_t* empty = full + 1;
  uint64_t* w_full = full + 2;

  const int warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) {
    mbar_init(full, 1);
    mbar_init(empty, 256);   // every consumer thread: its conv1 MMAs and its residual loads are done with the stage
    mbar_init(w_full, 1);
    fence_barrier_init();
  }
  __syncthreads();
  pdl_trigger();
  const int per_frame = tiles_x * tiles_y;

  if (warp == 0) {
    // ===================== TMA producer =====================
    if (elect_one()) {
      mbar_arrive_expect_tx(w_full, 2 * kWBytes);
      for (int off = 0; off < kWBytes; off += kTapBytes) {
        bulk_copy_g2s(sW1 + off, w1pack + off, kTapBytes, w_full);
        bulk_copy_g2s(sW2 + off, w2pack + off, kTapBytes, w_full);
      }
      pdl_wait();                             // weights are constants; activations must wait for the predecessor grids
      const uint64_t pol = l2_policy_stream();
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x, phase ^= 1) {
        const BlkTile tl(tile, tiles_x, per_frame, Cfg::kTW);
        mbar_wait(empty, phase ^ 1);
        mbar_arrive_expect_tx(full, Cfg::kStagePayload);
        tma_load_4d(sA, &tmap, full, 0, tl.x0 - 2, tl.y0 - 2, tl.n, pol);
      }
    }
  } else if (warp >= 4) {
    // ===================== consumers: both warpgroups work on every tile of the CTA =====================
    const int t = threadIdx.x & 127;
    const BlkThread th{(warp >> 2) - 1, t >> 5, t & 31};
    pdl_wait();                               // output writes must follow the predecessor grids
    mbar_wait(w_full, 0);
    float acc[Cfg::kN1 / 2], acc2[Cfg::kN2 / 2];
    uint32_t rv[Cfg::kG2][2];
    const int row0 = th.g * Cfg::kN1;          // this warpgroup's first conv1 row
    uint32_t phase = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x, phase ^= 1) {
      const uint32_t w1_base = opaque(smem_u32(sW1)), w2_base = opaque(smem_u32(sW2)), a_base = opaque(smem_u32(sA)),
                     mid_base = opaque(smem_u32(sMid));
      const float* b1p = opaque(bias1);
      const float* b2p = opaque(p.bias);
      const BlkTile tl(tile, tiles_x, per_frame, Cfg::kTW);
      mbar_wait(full, phase);
      conv1_issue<FOLD>(acc, a_base, w1_base, row0);
      load_residual<FOLD>(rv, a_base, th);    // while the MMAs run
      wgmma_wait<0>();
      mbar_arrive(empty);                     // the stage goes back to the producer: the next tile's load overlaps the rest
      consumers_bar_sync();                   // both warpgroups' conv2 of the previous tile has retired
      mid_epilogue<FOLD>(acc, mid_base, b1p, p, tl, th, row0);
      fence_proxy_async();                    // generic-proxy stores -> visible to wgmma
      consumers_bar_sync();
      conv2_issue<FOLD>(acc2, mid_base, w2_base, th.g);
      wgmma_wait<0>();
      out_epilogue<FOLD>(acc2, rv, b2p, p, tl, th);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
bool tc_block_supported(const ConvParams& p, bool fold) {
  if (p.in_dtype != B200ROMP_BF16 || p.out_dtype != B200ROMP_BF16 || p.res_dtype != B200ROMP_BF16) return false;
  if (p.cin != 64 || p.cout != 64 || p.up != 1 || p.out_nchw || p.pow_channel >= 0 || p.input_norm || !p.relu) return false;
  if (p.Hin != p.Hout || p.Win != p.Wout || p.Hout % 16 != 0 || p.Wout % (fold ? BlkCfg<true>::kTW : BlkCfg<false>::kTW) != 0) return false;
  if (p.in_C % 8 != 0 || p.in_c_off % 8 != 0 || p.out_C % 8 != 0 || p.out_c_off % 8 != 0) return false;
  // the residual is read from the staged input halo: it must be the block's input slice itself
  if (p.res != p.in || p.res_C != p.in_C || p.res_c_off != p.in_c_off || p.res_broadcast) return false;
  return (reinterpret_cast<uintptr_t>(p.in) & 15) == 0;
}

// one conv's weight image in shared-memory order.  Folded: the s = 0 taps as 128 B-row tiles, and of each s = -1 / s = +1
// tap only the 64 B-row chunk of the input channels its MMAs read (channels 32..63 = the second pixel of the pair for
// s = -1, channels 0..31 = the first for s = +1), at w_tap_off.
static int block_pack_weights(const float* w_oihw, bool fold, void** d_out, std::vector<void*>* allocs) {
  if (!fold) return tc_pack_weights(w_oihw, 64, 64, 9, 64, d_out, allocs, kRowB, 2);
  const std::vector<uint8_t> full = tc_pack_image(w_oihw, 64, 64, 9, 64, kRowB, 2);   // [tap][64 x 128 B]
  const std::vector<uint8_t> half = tc_pack_image(w_oihw, 64, 64, 9, 64, 64, 2);      // [tap][chunk][64 x 64 B]
  std::vector<uint8_t> img(BlkCfg<true>::kWBytes);
  for (int tap = 0; tap < 9; ++tap) {
    uint8_t* dst = img.data() + w_tap_off(true, tap);
    if (tap % 3 == 1) memcpy(dst, full.data() + (size_t)tap * kTapBytes, kTapBytes);
    else memcpy(dst, half.data() + (size_t)(2 * tap + (tap % 3 == 0 ? 1 : 0)) * kHalfTapBytes, kHalfTapBytes);
  }
  *d_out = upload(img.data(), img.size(), allocs);
  return *d_out ? B200ROMP_OK : B200ROMP_ECUDA;
}

int tc_block_prepare(const ConvParams& p, const float* w1_oihw, const float* b1, const float* w2_oihw, int sm_count,
                     TcConvPlan* plan, std::vector<void*>* allocs) {
  plan->kind = 60;
  plan->eb = 2;
  plan->cin = plan->cout = plan->nt = 64;
  plan->grid_x = sm_count;
  plan->grid_y = 1;
  plan->stages = 1;
  plan->smem_bytes = plan->fold ? BlkCfg<true>::kSmemBytes : BlkCfg<false>::kSmemBytes;
  int rc = block_pack_weights(w1_oihw, plan->fold, &plan->d_wpack, allocs);
  if (rc) return rc;
  rc = block_pack_weights(w2_oihw, plan->fold, &plan->d_wpack2, allocs);
  if (rc) return rc;
  plan->d_bias1 = static_cast<const float*>(upload(b1, 64 * sizeof(float), allocs));
  if (!plan->d_bias1) return B200ROMP_ECUDA;
  // the 64-channel input slice with a 20 x (TW + 4) halo box
  rc = tc_encode_nhwc_input(&plan->tmap_in, p, 2, 64, plan->fold ? BlkCfg<true>::kHaloW : BlkCfg<false>::kHaloW, kHaloH,
                            CU_TENSOR_MAP_SWIZZLE_128B, "conv_block_tc");
  if (rc) return rc;
  B2R_CUDA_OK(cudaFuncSetAttribute(conv_block_tc_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, BlkCfg<false>::kSmemBytes));
  B2R_CUDA_OK(cudaFuncSetAttribute(conv_block_tc_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, BlkCfg<true>::kSmemBytes));
  return B200ROMP_OK;
}

int tc_block_launch(const TcConvPlan& plan, const ConvParams& p, cudaStream_t stream) {
  const int tiles_x = p.Wout / (plan.fold ? BlkCfg<true>::kTW : BlkCfg<false>::kTW), tiles_y = p.Hout / 16;
  const int num_tiles = tiles_x * tiles_y * p.B;
  const dim3 grid(std::min(plan.grid_x, num_tiles));
  auto kern = plan.fold ? conv_block_tc_kernel<true> : conv_block_tc_kernel<false>;
  B2R_CUDA_OK(tc_launch(kern, grid, kBlkThreads, plan.smem_bytes, stream, plan.tmap_in, p, reinterpret_cast<const uint8_t*>(plan.d_wpack),
                        reinterpret_cast<const uint8_t*>(plan.d_wpack2), plan.d_bias1, tiles_x, tiles_y, num_tiles));
  return B200ROMP_OK;
}

}  // namespace b200romp
