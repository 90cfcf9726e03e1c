// Stem conv on wgmma: backbone.conv1 = Conv2d(3, 64, 3, stride 2, pad 1) + BN + ReLU on raw uint8 frames with the
// input normalisation x/255*2-1 folded in (simple_romp/romp/model.py:384-387).
//
// GEMM view: M = 128 output pixels (one 16x8 tile), N = 64, K = 27 taps*channels padded to 32 (two wgmma K=16 steps).
// The A tile cannot come straight from TMA (3-channel u8, stride 2).  A 3-D tensor map over the frames viewed as
// [N][H][W*3 bytes] brings the raw 33-row x 80-byte window of a tile into shared memory (zero fill outside the image,
// two windows in flight per producer warp = 8 per SM, so DRAM latency is hidden); the producer threads then convert:
// thread = output pixel reads its 27 bytes from the window and writes one 64-byte K-major row in the SWIZZLE_64B pattern
// the MMA descriptor expects (gathering the 27 bytes straight from global memory is latency-bound).
// Exactness: the operand is stored as (x - 127.5) in bf16 - exact for every integer 0..255 (8 significant bits) - and the
// weights carry the factor 2/255, so  sum w*(2/255)*(x-127.5) = sum w*(x/255*2-1)  and zero padding stays zero; the only
// rounding is the bf16 rounding of the scaled weights (same as every other layer on this engine).
// Warp roles (384 threads): warps 0-3 producers - each builds whole tiles in its private stage, so four gathers (one DRAM
// latency each) are in flight per SM; warpgroups 1 and 2 consume stages {0, 2} and {1, 3}: wgmma into registers, then the
// shared register epilogue (tc_device.cuh: bias + ReLU + bf16).
#include "conv_tc.cuh"
#include "tc_device.cuh"

namespace b200romp {

namespace {
constexpr int kStemStages = 4;                   // = producer warps, stage w is private to producer w
constexpr int kStemThreads = 384;                // warpgroup 0: producers, warpgroups 1-2: consumers
constexpr int kStemK = 32;                       // 27 padded to two wgmma K steps
constexpr int kStemRowB = kStemK * 2;            // 64 B rows -> SWIZZLE_64B
constexpr int kStemABytes = 128 * kStemRowB;     // 8 KB per stage
constexpr int kStemNT = 64;
constexpr int kStemBBytes = kStemNT * kStemRowB; // 4 KB weight image
constexpr int kRawRowB = 80;                     // bytes [6*x0 - 16, 6*x0 + 64) of each input row: 16 B aligned, covers ix = 2*x0-1 .. 2*x0+15
constexpr int kRawRows = 33;                     // iy = 2*y0 - 1 .. 2*y0 + 31
constexpr int kRawBytes = kRawRows * kRawRowB;   // 2640 B per window (TMA box)
constexpr int kRawStage = 2688;                  // padded to 128 B
constexpr int kRawDepth = 2;                     // windows in flight per producer warp
constexpr int kStemRawStride = kRawStage;
}  // namespace

__global__ void __launch_bounds__(kStemThreads, 1)
conv_stem_tc_kernel(const __grid_constant__ CUtensorMap raw_map, const ConvParams p, const uint8_t* __restrict__ wpack, int tiles_x,
                    int tiles_y, int num_tiles) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* sB = smem;
  uint8_t* sA = smem + kStemBBytes;
  uint8_t* raw_smem = sA + kStemStages * kStemABytes;
  uint64_t* full = reinterpret_cast<uint64_t*>(raw_smem + kStemStages * kRawDepth * kRawStage);
  uint64_t* empty = full + kStemStages;
  uint64_t* b_full = empty + kStemStages;
  uint64_t* raw_full = b_full + 1;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    for (int i = 0; i < kStemStages; ++i) {
      mbar_init(&full[i], 1);                    // its producer warp
      mbar_init(&empty[i], 4);                   // the 4 warps of the consuming warpgroup
    }
    mbar_init(b_full, 1);
    for (int i = 0; i < kStemStages * kRawDepth; ++i) mbar_init(&raw_full[i], 1);
    fence_barrier_init();
  }
  __syncthreads();
  const int per_frame = tiles_x * tiles_y;
  pdl_trigger();

  if (warp < kStemStages) {
    // ===================== im2col producers =====================
    const int pw = warp;                         // 0..3 = private stage
    if (threadIdx.x == 0) {
      mbar_arrive_expect_tx(b_full, kStemBBytes);
      bulk_copy_g2s(sB, wpack, kStemBBytes, b_full);
    }
    pdl_wait();                                  // frames may be produced by a predecessor kernel / copy
    const uint64_t pol = l2_policy_stream();
    uint8_t* a = sA + pw * kStemABytes;
    uint8_t* raw0 = raw_smem + pw * kRawDepth * kStemRawStride;
    uint64_t* rbar = raw_full + pw * kRawDepth;
    auto load_window = [&](int tile, int slot) {       // lane 0: raw input window of `tile` -> raw slot
      const int n = tile / per_frame, rem = tile % per_frame;
      const int y0 = (rem / tiles_x) * 16, x0 = (rem % tiles_x) * 8;
      mbar_arrive_expect_tx(&rbar[slot], kRawBytes);
      tma_load_3d(raw0 + slot * kStemRawStride, &raw_map, &rbar[slot], 6 * x0 - 16, 2 * y0 - 1, n, pol);
    };
    const int tstep = kStemStages * gridDim.x;
    const int first = blockIdx.x + pw * gridDim.x;
    if (lane == 0) {
#pragma unroll
      for (int d = 0; d < kRawDepth; ++d)
        if (first + d * tstep < num_tiles) load_window(first + d * tstep, d);
    }
    uint32_t phase = 0;
    int t_local = 0;
    for (int tile = first; tile < num_tiles; tile += tstep, ++t_local) {
      const int rem = tile % per_frame;
      const int y0 = (rem / tiles_x) * 16, x0 = (rem % tiles_x) * 8;
      const int slot = t_local % kRawDepth;
      const uint8_t* raw = raw0 + slot * kStemRawStride;
      mbar_wait(&rbar[slot], (uint32_t)(t_local / kRawDepth) & 1u);
      mbar_wait(&empty[pw], phase ^ 1);
#pragma unroll 2
      for (int j = 0; j < 4; ++j) {
        const int m = j * 32 + lane;                       // A row = pixel (m >> 3, m & 7) of the tile
        const int ty = m >> 3, px = m & 7;
        const int oy = y0 + ty, ox = x0 + px;
        uint32_t w[16];                                    // 32 bf16, k = r*9 + s*3 + c
        float v[32];
#pragma unroll
        for (int r = 0; r < 3; ++r) {
          const int iy = 2 * oy - 1 + r;
          const bool row_ok = iy >= 0 && iy < p.Hin;
          const uint8_t* src = raw + (2 * ty + r) * kRawRowB + 13 + 6 * px;    // byte of (iy, ix = 2*ox-1, c = 0)
#pragma unroll
          for (int s2 = 0; s2 < 3; ++s2) {
            const int ix = 2 * ox - 1 + s2;
            const bool ok = row_ok && ix >= 0 && ix < p.Win;
#pragma unroll
            for (int c = 0; c < 3; ++c) v[r * 9 + s2 * 3 + c] = ok ? (float)src[s2 * 3 + c] - 127.5f : 0.f;
          }
        }
#pragma unroll
        for (int k = 27; k < 32; ++k) v[k] = 0.f;
#pragma unroll
        for (int k = 0; k < 16; ++k) {
          __nv_bfloat162 h = __floats2bfloat162_rn(v[2 * k], v[2 * k + 1]);
          w[k] = *reinterpret_cast<uint32_t*>(&h);
        }
#pragma unroll
        for (int q4 = 0; q4 < 4; ++q4)                     // 16 B chunk q4 of row m, Swizzle<2,4,3>
          *reinterpret_cast<uint4*>(a + m * kStemRowB + ((q4 ^ ((m >> 1) & 3)) * 16)) = make_uint4(w[4 * q4], w[4 * q4 + 1], w[4 * q4 + 2], w[4 * q4 + 3]);
      }
      fence_proxy_async();                                 // generic-proxy writes -> visible to the tensor core
      __syncwarp();
      if (lane == 0) {
        mbar_arrive(&full[pw]);
        if (tile + kRawDepth * tstep < num_tiles) load_window(tile + kRawDepth * tstep, slot);   // window slot is free again
      }
      phase ^= 1;
    }
  } else {
    // ===================== consumers: warpgroup g takes the tiles of producers g and g + 2, in tile order =====================
    const int g = (warp >> 2) - 1, t = threadIdx.x & 127;
    pdl_wait();
    mbar_wait(b_full, 0);
    const uint32_t b_base = smem_u32(sB);
    int k_it = 0;
    for (int tile = blockIdx.x + g * gridDim.x; tile < num_tiles; tile += 2 * gridDim.x, ++k_it) {
      const int stage = g + 2 * (k_it & 1);
      const int n = tile / per_frame, rem = tile % per_frame;
      const int y0 = (rem / tiles_x) * 16, x0 = (rem % tiles_x) * 8;
      mbar_wait(&full[stage], (uint32_t)(k_it >> 1) & 1u);
      const uint32_t a_base = smem_u32(sA + stage * kStemABytes);
      float acc[2][kStemNT / 2];
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < kStemK / 16; ++k) {
        const uint64_t bdesc = make_smem_desc(b_base + k * 32, 8 * kStemRowB, kSw64);
        wgmma_any<kStemNT, 2>(acc[0], make_smem_desc(a_base + k * 32, 8 * kStemRowB, kSw64), bdesc, k);
        wgmma_any<kStemNT, 2>(acc[1], make_smem_desc(a_base + 64 * kStemRowB + k * 32, 8 * kStemRowB, kSw64), bdesc, k);
      }
      wgmma_commit();
      wgmma_wait<0>();
      if (lane == 0) mbar_arrive(&empty[stage]);
      wg_epilogue<kStemNT>(p, acc, p.bias, n, y0, x0, 0, t);
    }
  }
}

// ------------------------------------------------------------------------------------------------
bool tc_stem_supported(const ConvParams& p, int ksize, int stride) {
  return ksize == 3 && stride == 2 && p.cin == 3 && p.in_C == 3 && p.in_c_off == 0 && p.cout == 64 && p.in_dtype == B200ROMP_U8 &&
         p.input_norm && p.out_dtype == B200ROMP_BF16 && !p.out_nchw && p.up == 1 && p.res == nullptr && p.relu &&
         p.pow_channel < 0 && p.out_C == 64 && p.out_c_off == 0 && p.Hout % 16 == 0 && p.Wout % 8 == 0 &&
         p.Hout * 2 == p.Hin && p.Wout * 2 == p.Win && (p.Win * 3) % 16 == 0;
}

int tc_stem_prepare(const ConvParams& p, const float* w_oihw, int sm_count, TcConvPlan* plan, std::vector<void*>* allocs) {
  // weights as a 64 x 32 K-major matrix, k = r*9 + s*3 + c, scaled by 2/255 (the normalisation), zero padded
  std::vector<float> wk((size_t)64 * kStemK, 0.f);
  for (int co = 0; co < 64; ++co)
    for (int c = 0; c < 3; ++c)
      for (int r = 0; r < 3; ++r)
        for (int s = 0; s < 3; ++s)
          wk[(size_t)co * kStemK + r * 9 + s * 3 + c] = w_oihw[(((size_t)co * 3 + c) * 3 + r) * 3 + s] * (2.0f / 255.0f);
  int rc = tc_pack_weights(wk.data(), kStemK, 64, 1, kStemNT, &plan->d_wpack, allocs, kStemK * 2, 2);
  if (rc) return rc;
  plan->kind = 33;
  plan->cin = 3; plan->cout = 64; plan->nt = kStemNT; plan->stages = kStemStages;
  plan->grid_x = sm_count; plan->grid_y = 1;
  plan->smem_bytes = kStemBBytes + kStemStages * kStemABytes + kStemStages * kRawDepth * kRawStage + 2048;
  B2R_CUDA_OK(cudaFuncSetAttribute(conv_stem_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, plan->smem_bytes));
  return B200ROMP_OK;
}

int tc_stem_launch(const TcConvPlan& plan, const ConvParams& p, cudaStream_t stream) {
  // raw-window tensor map over the (caller-owned, re-bindable) u8 frames: [N][H][W*3 bytes], zero fill outside.  Encoded at
  // every launch, since the frames may be re-bound; a failure is reported as EINVAL, like the frame checks.
  B2R_REQUIRE((reinterpret_cast<uintptr_t>(p.in) & 15) == 0 && (p.Win * 3) % 16 == 0,
              "conv_stem_tc: frames must be 16 B aligned with a row pitch that is a multiple of 16 B");
  CUtensorMap raw;
  const cuuint64_t gdim[3] = {(cuuint64_t)p.Win * 3, (cuuint64_t)p.Hin, (cuuint64_t)p.B};
  const cuuint64_t gstr[2] = {(cuuint64_t)p.Win * 3, (cuuint64_t)p.Win * 3 * p.Hin};
  const cuuint32_t box[3] = {(cuuint32_t)kRawRowB, (cuuint32_t)kRawRows, 1};
  if (tc_encode_tiled(&raw, CU_TENSOR_MAP_DATA_TYPE_UINT8, 3, p.in, gdim, gstr, box, CU_TENSOR_MAP_SWIZZLE_NONE, "conv_stem_tc (frames)"))
    return B200ROMP_EINVAL;
  const int tiles_x = p.Wout / 8, tiles_y = p.Hout / 16;
  const int num_tiles = tiles_x * tiles_y * p.B;
  dim3 grid(std::min(plan.grid_x, num_tiles), 1);
  B2R_CUDA_OK(tc_launch(conv_stem_tc_kernel, grid, kStemThreads, plan.smem_bytes, stream, raw, p,
                        reinterpret_cast<const uint8_t*>(plan.d_wpack), tiles_x, tiles_y, num_tiles));
  return B200ROMP_OK;
}

}  // namespace b200romp
