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
// Geometry, per 16x8 output tile at (y0, x0) of frame n (pixel pairs when folded):
//   input stage: ONE TMA load of the 20x12 halo at (x0-2, y0-2), channels innermost, 128 B swizzle, zeros outside the
//            frame.  Halo pixel (hy, hx) is stage row hy*12 + hx.
//   conv1:   over a LINEAR domain: mid pixel (my, mx), my < 18, mx < 10, is GEMM row my*12 + mx, so tap (r, s) is the stage
//            shifted by r*12 + s rows and the 8-row groups are contiguous (SBO = 1024 B).  Rows 0..213 are needed, padded to
//            256 (4 m64 blocks): warpgroup g computes rows 128g..128g+127.  Columns 10, 11 of a mid row and rows >= 214 are
//            never read by conv2; the stage rows 240..281 TMA never writes feed only those.
//   mid:     relu(acc + b1) -> bf16, zero where the mid pixel lies outside the frame (the unfused conv2 reads TMA zero fill
//            there), stored to a 256 x 128 B buffer in the swizzled layout wgmma reads (16 B chunk ^ (row & 7)).
//   conv2:   the conv_tc.cu 3x3 mapping on the mid buffer: 8-pixel groups, SBO = 12 rows, tap (r, s) shifted by r*12 + s
//            rows.  Warpgroup g computes output tile rows 8g..8g+7 (one m64 x N = 64).
//   output:  (acc + b2) + x, ReLU, bf16.  x at the output pixels is the interior of the halo: read from shared memory
//            before the stage is handed back.
// Both convs keep the K order of conv_tc_kernel (taps 0..8 x 32-byte k-steps, the same folded halves skipped), so the fp32
// sums and therefore t and y are bit-identical to the unfused path.
//
// Shared memory: both convs' weights stay resident (2 x 72 KB), next to ONE input stage (36 KB) and the mid buffer (32 KB):
// 212 KB of the 227 KB.  With room for one stage only, both consumer warpgroups work on the same tile; the stage goes back to
// the producer once conv1 has retired, so the next tile's TMA load overlaps the mid epilogue, conv2 and the output epilogue.
#include "conv_tc.cuh"
#include "tc_device.cuh"

namespace b200romp {

namespace {

constexpr int kBlkThreads = 384;                        // warp 0 = TMA producer, warpgroups 1, 2 = consumers
constexpr int kRowB = 128;                              // one pixel row: 64 bf16 channels = one 128 B swizzle span
constexpr int kHaloW = 12, kHaloH = 20;                 // input halo of a 16x8 output tile, two 3x3 convs deep
constexpr int kTapBytes = 64 * kRowB;                   // one tap of one conv: 64 output x 64 input channels
constexpr int kWBytes = 9 * kTapBytes;
constexpr int kStagePayload = kHaloH * kHaloW * kRowB;  // what TMA writes: 240 rows
constexpr int kStageBytes = (282 * kRowB + 1023) / 1024 * 1024;   // + the rows 240..281 the padded mid rows read
constexpr int kMidBytes = 256 * kRowB;
constexpr int kSmemBytes = 2 * kWBytes + kStageBytes + kMidBytes + 1024 /*barriers*/ + 1024 /*align slack*/;
static_assert(kSmemBytes <= 227 * 1024, "fused block does not fit shared memory");

// the MMAs of a pixel-pair folded conv that only meet all-zero weights: first pixel (k-steps 0, 1) of the s = -1 taps,
// second pixel (k-steps 2, 3) of the s = +1 taps (net.cu fold_pixel_pairs, the kmask of the unfused path)
template <bool FOLD>
__device__ __forceinline__ constexpr bool blk_skip(int tap, int k) {
  return FOLD && ((tap % 3 == 0 && k < 2) || (tap % 3 == 2 && k >= 2));
}

// barrier over both consumer warpgroups (id 1; 0 is __syncthreads)
__device__ __forceinline__ void consumers_bar_sync() { asm volatile("bar.sync 1, 256;" ::: "memory"); }

__device__ __forceinline__ uint32_t ld_shared_b32(uint32_t addr) {
  uint32_t v;
  asm volatile("ld.shared.b32 %0, [%1];" : "=r"(v) : "r"(addr));
  return v;
}
__device__ __forceinline__ void st_shared_b32(uint32_t addr, uint32_t v) {
  asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(v) : "memory");
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

}  // namespace

template <bool FOLD>
__global__ void __launch_bounds__(kBlkThreads, 1)
conv_block_tc_kernel(const __grid_constant__ CUtensorMap tmap, const ConvParams p, const uint8_t* __restrict__ w1pack,
                     const uint8_t* __restrict__ w2pack, const float* __restrict__ bias1, int tiles_x, int tiles_y, int num_tiles) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* sW1 = smem;
  uint8_t* sW2 = smem + kWBytes;
  uint8_t* sA = smem + 2 * kWBytes;
  uint8_t* sMid = sA + kStageBytes;
  uint64_t* full = reinterpret_cast<uint64_t*>(sMid + kMidBytes);
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
      for (int t = 0; t < 9; ++t) {
        bulk_copy_g2s(sW1 + t * kTapBytes, w1pack + (size_t)t * kTapBytes, kTapBytes, w_full);
        bulk_copy_g2s(sW2 + t * kTapBytes, w2pack + (size_t)t * kTapBytes, kTapBytes, w_full);
      }
      pdl_wait();                             // weights are constants; activations must wait for the predecessor grids
      const uint64_t pol = l2_policy_stream();
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x, phase ^= 1) {
        const int n = tile / per_frame, rem = tile % per_frame;
        const int y0 = (rem / tiles_x) * 16, x0 = (rem % tiles_x) * 8;
        mbar_wait(empty, phase ^ 1);
        mbar_arrive_expect_tx(full, kStagePayload);
        tma_load_4d(sA, &tmap, full, 0, x0 - 2, y0 - 2, n, pol);
      }
    }
  } else if (warp >= 4) {
    // ===================== consumers: both warpgroups work on every tile of the CTA =====================
    const int g = (warp >> 2) - 1, t = threadIdx.x & 127, w = t >> 5, l = t & 31;
    pdl_wait();                               // output writes must follow the predecessor grids
    mbar_wait(w_full, 0);
    const int cl = 2 * (l & 3);               // this thread's channel pair inside each 8-channel group
    uint32_t phase = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x, phase ^= 1) {
      const uint32_t w1_base = opaque(smem_u32(sW1)), w2_base = opaque(smem_u32(sW2)), a_base = opaque(smem_u32(sA)),
                     mid_base = opaque(smem_u32(sMid));
      const float* b1p = opaque(bias1);
      const float* b2p = opaque(p.bias);
      const int n = tile / per_frame, rem = tile % per_frame;
      const int y0 = (rem / tiles_x) * 16, x0 = (rem % tiles_x) * 8;
      mbar_wait(full, phase);

      // ---- conv1: mid rows 128g .. 128g + 127 as two m64 blocks
      float acc[2][32];
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int j = 0; j < 32; ++j) acc[h][j] = 0.f;
      uint32_t scale_d = 0;
      wgmma_fence();
#pragma unroll
      for (int tap = 0; tap < 9; ++tap) {
        const uint32_t a_tap = a_base + (uint32_t)((128 * g + (tap / 3) * kHaloW + tap % 3) * kRowB);
        const uint32_t b_tap = w1_base + (uint32_t)(tap * kTapBytes);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          if (blk_skip<FOLD>(tap, k)) continue;
          const uint64_t bdesc = make_smem_desc(b_tap + k * 32, 8 * kRowB, kSw128);
          wgmma_n64(acc[0], make_smem_desc(a_tap + k * 32, 8 * kRowB, kSw128), bdesc, scale_d, false);
          wgmma_n64(acc[1], make_smem_desc(a_tap + 64 * kRowB + k * 32, 8 * kRowB, kSw128), bdesc, scale_d, false);
          scale_d = 1;
        }
      }
      wgmma_commit();
      // residual = the block input at this thread's output pixels (tile row 8g + 2w + e, column l / 4): halo pixel
      // (row + 2, column + 2), loaded while the MMAs run
      uint32_t rv[2][8];
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int hr = (8 * g + 2 * w + e + 2) * kHaloW + (l >> 2) + 2;
#pragma unroll
        for (int j = 0; j < 8; ++j) rv[e][j] = ld_shared_b32(a_base + hr * kRowB + ((j ^ (hr & 7)) << 4) + 2 * cl);
      }
      wgmma_wait<0>();
      mbar_arrive(empty);                     // the stage goes back to the producer: the next tile's load overlaps the rest

      // ---- mid epilogue: relu(acc + b1), zero outside the frame, bf16, swizzled into the mid buffer
      consumers_bar_sync();                   // both warpgroups' conv2 of the previous tile has retired
#pragma unroll
      for (int h = 0; h < 2; ++h) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int m = 64 * (2 * g + h) + 16 * w + (l >> 2) + 8 * e;
          const int my = m / kHaloW, mx = m % kHaloW;
          const bool inside = my < 18 && mx < 10 && (unsigned)(y0 - 1 + my) < (unsigned)p.Hout && (unsigned)(x0 - 1 + mx) < (unsigned)p.Wout;
          const uint32_t row = mid_base + m * kRowB;
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const int c = 8 * j + cl;
            float a = fmaxf(acc[h][4 * j + 2 * e] + __ldg(b1p + c), 0.f);
            float b = fmaxf(acc[h][4 * j + 2 * e + 1] + __ldg(b1p + c + 1), 0.f);
            if (!inside) a = b = 0.f;
            st_shared_b32(row + ((j ^ (m & 7)) << 4) + 2 * cl, pack_bf16x2(a, b));
          }
        }
      }
      fence_proxy_async();                    // generic-proxy stores -> visible to wgmma
      consumers_bar_sync();

      // ---- conv2: output tile rows 8g .. 8g + 7
      float acc2[32];
#pragma unroll
      for (int j = 0; j < 32; ++j) acc2[j] = 0.f;
      scale_d = 0;
      wgmma_fence();
#pragma unroll
      for (int tap = 0; tap < 9; ++tap) {
        const uint32_t a_tap = mid_base + (uint32_t)(((8 * g + tap / 3) * kHaloW + tap % 3) * kRowB);
        const uint32_t b_tap = w2_base + (uint32_t)(tap * kTapBytes);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          if (blk_skip<FOLD>(tap, k)) continue;
          wgmma_n64(acc2, make_smem_desc(a_tap + k * 32, kHaloW * kRowB, kSw128), make_smem_desc(b_tap + k * 32, 8 * kRowB, kSw128),
                    scale_d, false);
          scale_d = 1;
        }
      }
      wgmma_commit();
      wgmma_wait<0>();

      // ---- output epilogue: (acc + b2) + x, ReLU, bf16 (the order of the unfused conv2)
      __nv_bfloat16* out = reinterpret_cast<__nv_bfloat16*>(p.out);
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const size_t pix = ((size_t)n * p.Hout + y0 + 8 * g + 2 * w + e) * p.Wout + x0 + (l >> 2);
        __nv_bfloat162* o = reinterpret_cast<__nv_bfloat162*>(out + pix * p.out_C + p.out_c_off + cl);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const int c = 8 * j + cl;
          float a = acc2[4 * j + 2 * e] + __ldg(b2p + c), b = acc2[4 * j + 2 * e + 1] + __ldg(b2p + c + 1);
          const float2 r = res_pair(rv[e][j]);
          a += r.x; b += r.y;
          o[4 * j] = __floats2bfloat162_rn(fmaxf(a, 0.f), fmaxf(b, 0.f));
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
bool tc_block_supported(const ConvParams& p) {
  if (p.in_dtype != B200ROMP_BF16 || p.out_dtype != B200ROMP_BF16 || p.res_dtype != B200ROMP_BF16) return false;
  if (p.cin != 64 || p.cout != 64 || p.up != 1 || p.out_nchw || p.pow_channel >= 0 || p.input_norm || !p.relu) return false;
  if (p.Hin != p.Hout || p.Win != p.Wout || p.Hout % 16 != 0 || p.Wout % 8 != 0) return false;
  if (p.in_C % 8 != 0 || p.in_c_off % 8 != 0 || p.out_C % 8 != 0 || p.out_c_off % 8 != 0) return false;
  // the residual is read from the staged input halo: it must be the block's input slice itself
  if (p.res != p.in || p.res_C != p.in_C || p.res_c_off != p.in_c_off || p.res_broadcast) return false;
  return (reinterpret_cast<uintptr_t>(p.in) & 15) == 0;
}

int tc_block_prepare(const ConvParams& p, const float* w1_oihw, const float* b1, const float* w2_oihw, int sm_count,
                     TcConvPlan* plan, std::vector<void*>* allocs) {
  PFN_encodeTiled encode = tc_get_encode();
  if (!encode) {
    set_error("conv_block_tc: cuTensorMapEncodeTiled is unavailable");
    return B200ROMP_ECUDA;
  }
  plan->kind = 60;
  plan->eb = 2;
  plan->cin = plan->cout = plan->nt = 64;
  plan->grid_x = sm_count;
  plan->grid_y = 1;
  plan->stages = 1;
  plan->smem_bytes = kSmemBytes;
  int rc = tc_pack_weights(w1_oihw, 64, 64, 9, 64, &plan->d_wpack, allocs, kRowB, 2);
  if (rc) return rc;
  rc = tc_pack_weights(w2_oihw, 64, 64, 9, 64, &plan->d_wpack2, allocs, kRowB, 2);
  if (rc) return rc;
  void* db1 = nullptr;
  B2R_CUDA_OK(cudaMalloc(&db1, 64 * sizeof(float)));
  allocs->push_back(db1);
  B2R_CUDA_OK(cudaMemcpy(db1, b1, 64 * sizeof(float), cudaMemcpyHostToDevice));
  plan->d_bias1 = static_cast<const float*>(db1);
  // tensor map over the NHWC input slice: dims (C, W, H, N), 20x12 halo box, OOB -> zeros
  CUtensorMap tm;
  const cuuint64_t gdim[4] = {64, (cuuint64_t)p.Win, (cuuint64_t)p.Hin, (cuuint64_t)p.B};
  const cuuint64_t gstr[3] = {(cuuint64_t)p.in_C * 2, (cuuint64_t)p.Win * p.in_C * 2, (cuuint64_t)p.Hin * p.Win * p.in_C * 2};
  const cuuint32_t box[4] = {64, kHaloW, kHaloH, 1};
  const cuuint32_t estr[4] = {1, 1, 1, 1};
  void* base = const_cast<uint8_t*>(static_cast<const uint8_t*>(p.in) + (size_t)p.in_c_off * 2);
  CUresult cr = encode(&tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, base, gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                       CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (cr != CUDA_SUCCESS) {
    set_error("conv_block_tc: cuTensorMapEncodeTiled failed with %d", (int)cr);
    return B200ROMP_ECUDA;
  }
  memcpy(plan->tmap_in, &tm, sizeof(tm));
  B2R_CUDA_OK(cudaFuncSetAttribute(conv_block_tc_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytes));
  B2R_CUDA_OK(cudaFuncSetAttribute(conv_block_tc_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytes));
  return B200ROMP_OK;
}

int tc_block_launch(const TcConvPlan& plan, const ConvParams& p, cudaStream_t stream) {
  CUtensorMap tm;
  memcpy(&tm, plan.tmap_in, sizeof(tm));
  const int tiles_x = p.Wout / 8, tiles_y = p.Hout / 16;
  const int num_tiles = tiles_x * tiles_y * p.B;
  const dim3 grid(std::min(plan.grid_x, num_tiles));
  auto kern = plan.fold ? conv_block_tc_kernel<true> : conv_block_tc_kernel<false>;
  B2R_CUDA_OK(tc_launch(kern, grid, kBlkThreads, plan.smem_bytes, stream, tm, p, reinterpret_cast<const uint8_t*>(plan.d_wpack),
                        reinterpret_cast<const uint8_t*>(plan.d_wpack2), plan.d_bias1, tiles_x, tiles_y, num_tiles));
  return B200ROMP_OK;
}

}  // namespace b200romp
