// Fused ResNet Bottleneck on the wgmma engine: y = relu(W3 relu(W2 * relu(W1 x + b1) + b2) + b3 + x), 1x1 256 -> 64,
// 3x3 stride 1 64 -> 64, 1x1 64 -> 256, bf16 NHWC, one kernel per block (HRNet layer1.1 .. layer1.3).
//
// Unfused, the three convs move eight activation passes of 2..8 channel-groups through HBM (x is read by conv1 and again as
// conv3's residual, t1 and t2 are written and read back): 2,048 MiB per block at batch 64 and 128 x 128.  Here t1 and t2
// live only in shared memory, so a block reads x once from HBM and writes y once: half the bytes of a layer that is bound by
// them.  The residual is re-read from L2 right after the tile's halo was loaded.
//
// Geometry, per 16x8 output tile at (y0, x0) of frame n:
//   x stages: the 18x10 halo at (x0-1, y0-1) arrives by TMA in four 64-channel chunks (128 B swizzle, zeros outside the
//            frame) through a ring of two stages, so the next tile's first two chunks load during conv2, conv3 and the
//            epilogues.  Halo pixel (hy, hx) is stage row hy*10 + hx.
//   conv1:   1x1 over the LINEAR halo domain: mid pixel (my, mx) is GEMM row my*10 + mx; rows 0..179, padded to 192 (three
//            m64 blocks).  Warpgroup g computes block g at N = 64 and output channels 32g..32g+31 of block 2 at N = 32.
//            Rows 180..191 read stage rows TMA never writes and feed mid rows conv2 never reads.
//   mid:     relu(acc + b1) -> bf16, zero where the mid pixel lies outside the frame (the unfused conv2 reads TMA zero fill
//            there), stored to a 192 x 128 B buffer in the swizzled layout wgmma reads (16 B chunk ^ (row & 7)).
//   conv2:   the conv_tc.cu 3x3 mapping on the mid buffer: 8-pixel groups, SBO = 10 rows, tap (r, s) shifted by r*10 + s
//            rows.  Warpgroup g computes output tile rows 8g..8g+7 (one m64, N = 64).
//   t2:      relu(acc + b2) -> bf16 into a 128 x 128 B swizzled buffer; warpgroup g writes and later reads only rows 64g..
//   conv3:   1x1 on t2 at N = 256 as two m64n128 passes per warpgroup (64 accumulator registers each).
//   output:  (acc + b3) + x, ReLU, bf16; the residual x is loaded while the pass's MMAs run.
// STORE_MIDS (a net where other ops also read t1 or t2): the tile's interior of t1 and its t2 are written to HBM as well,
// each where its pointer is set, as the per-conv path would write them.
// Every conv keeps the K order of conv_tc_kernel (conv1: 4 chunks x 4 k-steps, conv2: taps 0..8 x 4 k-steps, conv3: 4
// k-steps) and every epilogue its arithmetic order, so t1, t2 and y are bit-identical to the unfused path.
#include "conv_tc.cuh"
#include "tc_device.cuh"

namespace b200romp {

namespace {

constexpr int kBnThreads = 384;                         // warp 0 = TMA producer, warpgroups 1, 2 = consumers
constexpr int kRowB = 128;                              // one pixel row of one 64-channel chunk: one 128 B swizzle span
constexpr int kHaloW = 10, kHaloH = 18;                 // input halo of a 16x8 output tile, one 3x3 conv deep
constexpr int kChunks = 4;                              // 256 input channels = 4 chunks of 64
constexpr int kRing = 2;                                // x stages
constexpr int kW1Bytes = kChunks * 64 * kRowB;          // [chunk][64 out][64 in]
constexpr int kW2Bytes = 9 * 64 * kRowB;                // [tap][64 out][64 in]
constexpr int kW3Bytes = 256 * kRowB;                   // [256 out][64 in]
constexpr int kStagePayload = kHaloH * kHaloW * kRowB;  // what TMA writes: 180 rows
constexpr int kStageBytes = 192 * kRowB;                // + the rows 180..191 the padded conv1 block reads
constexpr int kMidBytes = 192 * kRowB;
constexpr int kT2Bytes = 128 * kRowB;
constexpr int kSmemBytes = kW1Bytes + kW2Bytes + kW3Bytes + kRing * kStageBytes + kMidBytes + kT2Bytes + 1024 /*barriers*/ +
                           1024 /*align slack*/;
static_assert(kSmemBytes <= 227 * 1024, "fused bottleneck does not fit shared memory");

// barrier over both consumer warpgroups (id 1; 0 is __syncthreads); ids 2, 3: one consumer warpgroup
__device__ __forceinline__ void consumers_bar_sync() { asm volatile("bar.sync 1, 256;" ::: "memory"); }

__device__ __forceinline__ void st_shared_b32(uint32_t addr, uint32_t v) {
  asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(v) : "memory");
}
// an opaque copy: keeps the compiler from hoisting everything derived from a loop-invariant value (the shared-memory
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

template <bool STORE_MIDS>
__global__ void __launch_bounds__(kBnThreads, 1)
conv_bottleneck_tc_kernel(const __grid_constant__ CUtensorMap tmap, const ConvParams p, const uint8_t* __restrict__ w1pack,
                          const uint8_t* __restrict__ w2pack, const uint8_t* __restrict__ w3pack, const float* __restrict__ bias1,
                          const float* __restrict__ bias2, BottleneckMids mids, int tiles_x, int tiles_y, int num_tiles) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* sW1 = smem;
  uint8_t* sW2 = sW1 + kW1Bytes;
  uint8_t* sW3 = sW2 + kW2Bytes;
  uint8_t* sA = sW3 + kW3Bytes;
  uint8_t* sMid = sA + kRing * kStageBytes;
  uint8_t* sT2 = sMid + kMidBytes;
  uint64_t* full = reinterpret_cast<uint64_t*>(sT2 + kT2Bytes);
  uint64_t* empty = full + kRing;
  uint64_t* w_full = empty + kRing;

  const int warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) {
    for (int i = 0; i < kRing; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], 8);   // one arrival per consumer warp: both warpgroups read every stage
    }
    mbar_init(w_full, 1);
    fence_barrier_init();
  }
  __syncthreads();
  pdl_trigger();
  const int per_frame = tiles_x * tiles_y;

  if (warp == 0) {
    // ===================== TMA producer =====================
    if (elect_one()) {
      mbar_arrive_expect_tx(w_full, kW1Bytes + kW2Bytes + kW3Bytes);
      bulk_copy_g2s(sW1, w1pack, kW1Bytes, w_full);
      for (int t = 0; t < 9; ++t) bulk_copy_g2s(sW2 + t * 64 * kRowB, w2pack + (size_t)t * 64 * kRowB, 64 * kRowB, w_full);
      bulk_copy_g2s(sW3, w3pack, kW3Bytes, w_full);
      pdl_wait();                             // weights are constants; activations must wait for the predecessor grids
      const uint64_t pol = l2_policy_stream();
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int n = tile / per_frame, rem = tile % per_frame;
        const int y0 = (rem / tiles_x) * 16, x0 = (rem % tiles_x) * 8;
        for (int c = 0; c < kChunks; ++c) {
          mbar_wait(&empty[stage], phase ^ 1);
          mbar_arrive_expect_tx(&full[stage], kStagePayload);
          tma_load_4d(sA + stage * kStageBytes, &tmap, &full[stage], c * 64, x0 - 1, y0 - 1, n, pol);
          if (++stage == kRing) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else if (warp >= 4) {
    // ===================== consumers: both warpgroups work on every tile of the CTA =====================
    const int g = (warp >> 2) - 1, t = threadIdx.x & 127, w = t >> 5, l = t & 31;
    pdl_wait();                               // residual reads / output writes must follow the predecessor grids
    mbar_wait(w_full, 0);
    const int cl = 2 * (l & 3);               // this thread's channel pair inside each 8-channel group
    int stage = 0;
    uint32_t phase = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      const uint32_t w1_base = opaque(smem_u32(sW1)), w2_base = opaque(smem_u32(sW2)), w3_base = opaque(smem_u32(sW3)),
                     a_base = opaque(smem_u32(sA)), mid_base = opaque(smem_u32(sMid)), t2_base = opaque(smem_u32(sT2));
      const float* b1p = opaque(bias1);
      const float* b2p = opaque(bias2);
      const float* b3p = opaque(p.bias);
      const int n = tile / per_frame, rem = tile % per_frame;
      const int y0 = (rem / tiles_x) * 16, x0 = (rem % tiles_x) * 8;

      // ---- conv1: mid rows 64g .. 64g + 63 at N = 64, rows 128 .. 191 x channels 32g .. 32g + 31 at N = 32
      float acc[32], acc_b[16];
#pragma unroll
      for (int j = 0; j < 32; ++j) acc[j] = 0.f;
#pragma unroll
      for (int j = 0; j < 16; ++j) acc_b[j] = 0.f;
      uint32_t scale_d = 0;
      int prev = -1;
#pragma unroll
      for (int c = 0; c < kChunks; ++c) {
        mbar_wait(&full[stage], phase);
        const uint32_t a_st = a_base + (uint32_t)(stage * kStageBytes);
        const uint32_t b_ch = w1_base + (uint32_t)(c * 64 * kRowB);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          wgmma_n64(acc, make_smem_desc(a_st + 64 * g * kRowB + k * 32, 8 * kRowB, kSw128),
                    make_smem_desc(b_ch + k * 32, 8 * kRowB, kSw128), scale_d, false);
          wgmma_n32(acc_b, make_smem_desc(a_st + 128 * kRowB + k * 32, 8 * kRowB, kSw128),
                    make_smem_desc(b_ch + 32 * g * kRowB + k * 32, 8 * kRowB, kSw128), scale_d, false);
          scale_d = 1;
        }
        wgmma_commit();
        if (prev >= 0) {                      // the previous chunk's MMAs have retired: its stage goes back to the producer
          wgmma_wait<1>();
          if (l == 0) mbar_arrive(&empty[prev]);
        }
        prev = stage;
        if (++stage == kRing) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      if (l == 0) mbar_arrive(&empty[prev]);

      // ---- mid epilogue: relu(acc + b1), zero outside the frame, bf16, swizzled into the mid buffer
      consumers_bar_sync();                   // both warpgroups' conv2 of the previous tile has retired
      auto mid_store = [&](int m, int j, float a, float b) {   // mid row m, 8-channel group j
        const int my = m / kHaloW, mx = m % kHaloW;
        const bool inside = my < kHaloH && (unsigned)(y0 - 1 + my) < (unsigned)p.Hout && (unsigned)(x0 - 1 + mx) < (unsigned)p.Wout;
        if (!inside) a = b = 0.f;
        const uint32_t v = pack_bf16x2(a, b);
        st_shared_b32(mid_base + m * kRowB + ((j ^ (m & 7)) << 4) + 2 * cl, v);
        if constexpr (STORE_MIDS) {   // t1 at the tile's own pixels (the halo ring belongs to the neighbouring tiles)
          if (mids.t1 != nullptr && my >= 1 && my <= 16 && mx >= 1 && mx <= 8) {
            const size_t pix = ((size_t)n * p.Hout + y0 - 1 + my) * p.Wout + x0 - 1 + mx;
            *reinterpret_cast<uint32_t*>(mids.t1 + pix * mids.t1_C + 8 * j + cl) = v;
          }
        }
      };
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int m = 64 * g + 16 * w + (l >> 2) + 8 * e;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const int c = 8 * j + cl;
          mid_store(m, j, fmaxf(acc[4 * j + 2 * e] + __ldg(b1p + c), 0.f), fmaxf(acc[4 * j + 2 * e + 1] + __ldg(b1p + c + 1), 0.f));
        }
        const int mb = 128 + 16 * w + (l >> 2) + 8 * e;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int c = 32 * g + 8 * j + cl;
          mid_store(mb, 4 * g + j, fmaxf(acc_b[4 * j + 2 * e] + __ldg(b1p + c), 0.f),
                    fmaxf(acc_b[4 * j + 2 * e + 1] + __ldg(b1p + c + 1), 0.f));
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
        const uint32_t b_tap = w2_base + (uint32_t)(tap * 64 * kRowB);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          wgmma_n64(acc2, make_smem_desc(a_tap + k * 32, kHaloW * kRowB, kSw128), make_smem_desc(b_tap + k * 32, 8 * kRowB, kSw128),
                    scale_d, false);
          scale_d = 1;
        }
      }
      wgmma_commit();
      wgmma_wait<0>();

      // ---- t2 epilogue: relu(acc + b2), bf16, into this warpgroup's t2 rows (tile pixel m = 64g + 16w + l/4 + 8e)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int m = 64 * g + 16 * w + (l >> 2) + 8 * e;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const int c = 8 * j + cl;
          const uint32_t v = pack_bf16x2(fmaxf(acc2[4 * j + 2 * e] + __ldg(b2p + c), 0.f), fmaxf(acc2[4 * j + 2 * e + 1] + __ldg(b2p + c + 1), 0.f));
          st_shared_b32(t2_base + m * kRowB + ((j ^ (m & 7)) << 4) + 2 * cl, v);
          if constexpr (STORE_MIDS) {
            if (mids.t2 != nullptr) {
              const size_t pix = ((size_t)n * p.Hout + y0 + 8 * g + 2 * w + e) * p.Wout + x0 + (l >> 2);
              *reinterpret_cast<uint32_t*>(mids.t2 + pix * mids.t2_C + c) = v;
            }
          }
        }
      }
      fence_proxy_async();
      wg_bar_sync(2 + g);

      // ---- conv3 + output epilogue, output channels 128h .. 128h + 127 per pass: (acc + b3) + x, ReLU, bf16
      const __nv_bfloat16* res = reinterpret_cast<const __nv_bfloat16*>(p.res);
      __nv_bfloat16* out = reinterpret_cast<__nv_bfloat16*>(p.out);
#pragma unroll 1
      for (int h = 0; h < 2; ++h) {
        float acc3[64];
#pragma unroll
        for (int j = 0; j < 64; ++j) acc3[j] = 0.f;
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k)
          wgmma_n128_bf16(acc3, make_smem_desc(t2_base + 64 * g * kRowB + k * 32, 8 * kRowB, kSw128),
                          make_smem_desc(w3_base + h * 128 * kRowB + k * 32, 8 * kRowB, kSw128), k > 0 ? 1u : 0u);
        wgmma_commit();
        // this thread's output pixels: tile row 8g + 2w + e, column l / 4
        uint32_t rv[2][16];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const size_t pix = ((size_t)n * p.Hout + y0 + 8 * g + 2 * w + e) * p.Wout + x0 + (l >> 2);
          const uint32_t* r = reinterpret_cast<const uint32_t*>(res + pix * p.res_C + p.res_c_off + 128 * h + cl);
#pragma unroll
          for (int j = 0; j < 16; ++j) rv[e][j] = r[4 * j];
        }
        wgmma_wait<0>();
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const size_t pix = ((size_t)n * p.Hout + y0 + 8 * g + 2 * w + e) * p.Wout + x0 + (l >> 2);
          __nv_bfloat162* o = reinterpret_cast<__nv_bfloat162*>(out + pix * p.out_C + p.out_c_off + 128 * h + cl);
#pragma unroll
          for (int j = 0; j < 16; ++j) {
            const int c = 128 * h + 8 * j + cl;
            float a = acc3[4 * j + 2 * e] + __ldg(b3p + c), b = acc3[4 * j + 2 * e + 1] + __ldg(b3p + c + 1);
            const float2 r = res_pair(rv[e][j]);
            a += r.x; b += r.y;
            o[4 * j] = __floats2bfloat162_rn(fmaxf(a, 0.f), fmaxf(b, 0.f));
          }
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
bool tc_bottleneck_supported(const ConvParams& p) {
  if (p.in_dtype != B200ROMP_BF16 || p.out_dtype != B200ROMP_BF16 || p.res_dtype != B200ROMP_BF16) return false;
  if (p.cin != 256 || p.cout != 256 || p.up != 1 || p.out_nchw || p.pow_channel >= 0 || p.input_norm || !p.relu) return false;
  if (p.Hin != p.Hout || p.Win != p.Wout || p.Hout % 16 != 0 || p.Wout % 8 != 0) return false;
  if (p.in_C % 8 != 0 || p.in_c_off % 8 != 0 || p.out_C % 8 != 0 || p.out_c_off % 8 != 0) return false;
  // the residual is the block's input slice itself, at the output pixels
  if (p.res != p.in || p.res_C != p.in_C || p.res_c_off != p.in_c_off || p.res_broadcast) return false;
  return (reinterpret_cast<uintptr_t>(p.in) & 15) == 0;
}

int tc_bottleneck_prepare(const ConvParams& p, const float* w1_oihw, const float* b1, const float* w2_oihw, const float* b2,
                          const float* w3_oihw, int sm_count, TcConvPlan* plan, std::vector<void*>* allocs) {
  plan->kind = 70;
  plan->eb = 2;
  plan->cin = plan->cout = 256;
  plan->nt = 256;
  plan->grid_x = sm_count;
  plan->grid_y = 1;
  plan->stages = kRing;
  plan->smem_bytes = kSmemBytes;
  int rc = tc_pack_weights(w1_oihw, 256, 64, 1, 64, &plan->d_wpack, allocs, kRowB, 2);   // [chunk][64 x 128 B]
  if (!rc) rc = tc_pack_weights(w2_oihw, 64, 64, 9, 64, &plan->d_wpack2, allocs, kRowB, 2);
  if (!rc) rc = tc_pack_weights(w3_oihw, 64, 256, 1, 256, &plan->d_wpack3, allocs, kRowB, 2);
  if (rc) return rc;
  plan->d_bias1 = static_cast<const float*>(upload(b1, 64 * sizeof(float), allocs));
  plan->d_bias2 = static_cast<const float*>(upload(b2, 64 * sizeof(float), allocs));
  if (!plan->d_bias1 || !plan->d_bias2) return B200ROMP_ECUDA;
  // the 256-channel input slice, loaded 64 channels at a time with a 10 x 18 halo box
  rc = tc_encode_nhwc_input(&plan->tmap_in, p, 2, 64, kHaloW, kHaloH, CU_TENSOR_MAP_SWIZZLE_128B, "conv_bottleneck_tc");
  if (rc) return rc;
  B2R_CUDA_OK(cudaFuncSetAttribute(conv_bottleneck_tc_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytes));
  B2R_CUDA_OK(cudaFuncSetAttribute(conv_bottleneck_tc_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytes));
  return B200ROMP_OK;
}

int tc_bottleneck_launch(const TcConvPlan& plan, const ConvParams& p, const BottleneckMids& mids, cudaStream_t stream) {
  const int tiles_x = p.Wout / 8, tiles_y = p.Hout / 16;
  const int num_tiles = tiles_x * tiles_y * p.B;
  const dim3 grid(std::min(plan.grid_x, num_tiles));
  auto kern = mids.t1 != nullptr || mids.t2 != nullptr ? conv_bottleneck_tc_kernel<true> : conv_bottleneck_tc_kernel<false>;
  B2R_CUDA_OK(tc_launch(kern, grid, kBnThreads, plan.smem_bytes, stream, plan.tmap_in, p, reinterpret_cast<const uint8_t*>(plan.d_wpack),
                        reinterpret_cast<const uint8_t*>(plan.d_wpack2), reinterpret_cast<const uint8_t*>(plan.d_wpack3),
                        plan.d_bias1, plan.d_bias2, mids, tiles_x, tiles_y, num_tiles));
  return B200ROMP_OK;
}

}  // namespace b200romp
