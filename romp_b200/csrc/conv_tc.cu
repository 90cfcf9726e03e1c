// wgmma implicit-GEMM convolution engine for sm_90a (the dominant kernel of the hot path).
//
// Replaces, per layer, cuDNN Conv2d + separate BatchNorm/ReLU/add/Upsample kernels of the reference
// (simple_romp/romp/model.py:49-123,185-244) for 1x1, 3x3 stride-1 and 3x3 stride-2 convolutions with
// Cin in {32,64,128,256} on NHWC bf16 activations (fp32 accumulate), or on fp32 activations consumed as TF32.
//
// Mapping (im2col-free):
//   GEMM M = 128 output pixels = one 16x8 spatial tile of one frame (two wgmma m64 halves: tile rows 0-7 / 8-15)
//   GEMM N = NT output channels (64, 32, or 16 for the TF32 3x3 256-channel layers) per CTA, weights RESIDENT in shared memory for the CTA's lifetime (persistent
//            CTAs loop over pixel tiles)
//   GEMM K = taps x Cin, walked as (channel chunk) x (tap) x (32-byte wgmma K step)
//   A operand, stride 1: ONE TMA load per (tile, chunk) brings the (16+2)x(8+2) halo tile, channels innermost,
//            hardware-swizzled (128B, or 64B for 64-byte rows).  The 9 taps are 9 *shifted shared-memory descriptors*
//            into that same halo tile: start address + (r*10+s) pixel rows, stride-byte-offset = 10 pixel rows (one image
//            row of the halo), so the input is read from L2 once, not 9 times.  Zero padding comes from TMA out-of-bounds
//            fill (negative start coordinates).
//   A operand, stride 2: a stride-2 3x3 conv on X[H,W,C] is a 2x2-tap stride-1 conv on the space-to-depth view
//            X'[H/2,W/2,(ph,pw,C)]: input row 2*oy+r-1 is (hh,ph) = (oy-1,1), (oy,0), (oy,1) for r = 0,1,2 (same for
//            columns).  A 5-D tensor map (dims: [pw*C+c], ww, ph, hh, n) addresses the NHWC tensor, so nothing is
//            rearranged in HBM; per (tile, chunk) the producer issues 4 loads - one per input parity - of (17|16)x(9|8)
//            sub-tiles, and tap (r,s) is a shifted descriptor into sub-tile (ph = r!=1, pw = s!=1).
//   D: fp32 accumulators in the registers of the consumer warpgroup; the epilogue (bias, residual, ReLU, upsample, dtype,
//            NCHW maps) runs straight from those registers.
// Warp roles (384 threads): warp 0 = TMA producer (one elected thread), warpgroups 1 and 2 = consumers.  Each consumer owns
//            a private ring of pipeline stages and takes every other tile of the CTA, so one warpgroup's epilogue overlaps
//            the other's MMAs.  Launched with programmatic dependent launch (prologue overlaps the previous conv's tail).
// SWAP (plan kind 31: bf16 3x3 stride 1, 128 -> 128 channels, bf16 NHWC output): the operands trade places.  The resident
//            weight slab is A (M = the CTA's 64 output channels; the same image and descriptors as B above) and the 16x8
//            pixel tile is B (N = 128: its 16 8-pixel groups are halo rows SBO apart, so each tap is the shifted descriptor
//            of the A operand above, now spanning both halves).  One m64n128k16 reads 2 + 4 KB of shared memory where the
//            two m64n64k16 read 8 KB.  Chunks, taps and k-steps run in the same order, so the fp32 sums are bit-identical
//            (tools/wgmma_swap_probe.cu); the accumulators come out channel-major and go through wg_epilogue_swap.
#include <mutex>

#include "conv_tc.cuh"
#include "tc_device.cuh"

namespace b200romp {

thread_local int g_tc_pdl_override = -1;

constexpr int kTcThreads = 384;
constexpr int kMaxRings = 2;

// bytes per pixel row of a stride-2 stage: half rows (64 B) once a full row would leave a single pipeline stage next to the
// resident weights (bf16 Cin = 256: 147 KB of weights + 74 KB per 128 B-row stage)
__host__ __device__ constexpr int s2_row_bytes(int cin, int eb) { return cin * eb >= 512 ? 64 : (cin * eb < 128 ? cin * eb : 128); }

// the smem stages are split into one private ring per consumer warpgroup: ring 0 gets the larger half.  With fewer than 4
// stages (weight-heavy layers) a split would leave one stage per ring, i.e. no overlap of a ring's TMA load with its MMAs;
// then one consumer owns all stages.
__host__ __device__ constexpr int tc_num_rings(int stages) { return stages >= 4 ? kMaxRings : 1; }
__host__ __device__ constexpr int tc_ring_size(int stages, int ring) { return tc_num_rings(stages) == 1 ? stages : (stages + 1 - ring) / 2; }
__host__ __device__ constexpr int tc_ring_base(int stages, int ring) { return ring ? (stages + 1) / 2 : 0; }

// MODE: 1 = 1x1, 3 = 3x3 stride 1, 2 = 3x3 stride 2
template <int MODE, int CIN, int NT, int EB>
struct TcCfg {
  static constexpr bool S2 = MODE == 2;
  static constexpr int KS = MODE == 1 ? 1 : 3;
  static constexpr int TAPS = KS * KS;
  static constexpr int PAD = KS / 2;
  static constexpr int ROWB = S2 ? s2_row_bytes(CIN, EB) : tc_row_bytes(KS, CIN, EB);
  static constexpr int CW = ROWB / EB;
  static constexpr int KCH = CIN / CW;
  static constexpr int KSTEPS = ROWB / 32;   // wgmma K steps (32 B = 16 bf16 / 8 tf32) per row
  static constexpr uint32_t LAYOUT = tc_layout(ROWB);
  static constexpr int HW_ = 8 + 2 * PAD;    // stride 1: halo tile
  static constexpr int HH = 16 + 2 * PAD;
  // stride 2: sub-tile i = (ph ? 0 : 2) + (pw ? 0 : 1):  (1,1) 17x9, (1,0) 17x8, (0,1) 16x9, (0,0) 16x8
  __host__ __device__ static constexpr int BH(int i) { return i < 2 ? 17 : 16; }
  __host__ __device__ static constexpr int BW(int i) { return (i & 1) ? 8 : 9; }
  __host__ __device__ static constexpr int SUB_BYTES(int i) { return (BH(i) * BW(i) * ROWB + 1023) / 1024 * 1024; }
  __host__ __device__ static constexpr int SUB_OFF(int i) { return i == 0 ? 0 : SUB_OFF(i - 1) + SUB_BYTES(i - 1); }
  static constexpr int STAGE_PAYLOAD = S2 ? (17 * 9 + 17 * 8 + 16 * 9 + 16 * 8) * ROWB : HH * HW_ * ROWB;
  static constexpr int STAGE_BYTES = S2 ? SUB_OFF(3) + SUB_BYTES(3) : (STAGE_PAYLOAD + 1023) / 1024 * 1024;
  static constexpr int BTILE = NT * ROWB;
  static constexpr int B_BYTES = TAPS * KCH * BTILE;
  // the one shape a pixel-pair folded 32->32 layer runs as (net.cu fold_pixel_pairs): only it reads kmask, a data-dependent
  // branch between wgmmas costs the other instantiations their MMA overlap
  static constexpr bool FOLDABLE = MODE == 3 && CIN == 64 && NT == 64 && EB == 2;
};

// kmask: bit (tap * 2 + half) = 0 skips the MMAs of that channel half of that tap (all-zero weights of a pixel-pair folded
// conv, see net.cu fold_pixel_pairs; single-chunk layers only).  GENERIC: outputs that are not NHWC at conv resolution with
// whole channel tiles (NCHW maps, 1.1**x, upsampling); the other variant has only the NHWC epilogue (see wg_epilogue).
template <int MODE, int CIN, int NT, int EB, bool GENERIC, bool SWAP = false>
__global__ void __launch_bounds__(kTcThreads, 1)
conv_tc_kernel(const __grid_constant__ CUtensorMap tmap, const __grid_constant__ S2Maps s2maps, const ConvParams p,
               const uint8_t* __restrict__ wpack, int tiles_x, int tiles_y, int num_tiles, int stages, unsigned kmask) {
  using Cfg = TcCfg<MODE, CIN, NT, EB>;
  static_assert(!SWAP || (MODE == 3 && NT == 64 && EB == 2 && !GENERIC), "the swapped plan is bf16 3x3 stride 1, NHWC, M = 64");
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* sB = smem;
  uint8_t* sA = smem + Cfg::B_BYTES;
  uint64_t* full = reinterpret_cast<uint64_t*>(sA + (size_t)stages * Cfg::STAGE_BYTES);
  uint64_t* empty = full + stages;
  uint64_t* b_full = empty + stages;

  const int warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) {
    for (int i = 0; i < stages; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], 4);   // one arrival per warp of the consuming warpgroup
    }
    mbar_init(b_full, 1);
    fence_barrier_init();
  }
  __syncthreads();
  pdl_trigger();
  const int per_frame = tiles_x * tiles_y;
  const int nrings = tc_num_rings(stages);   // consumer warpgroups in use = private stage rings

  if (warp == 0) {
    // ===================== TMA producer =====================
    if (elect_one()) {
      mbar_arrive_expect_tx(b_full, Cfg::B_BYTES);
      const uint8_t* wsrc = wpack + (size_t)blockIdx.y * Cfg::B_BYTES;
      for (int i = 0; i < Cfg::TAPS * Cfg::KCH; ++i)
        bulk_copy_g2s(sB + (size_t)i * Cfg::BTILE, wsrc + (size_t)i * Cfg::BTILE, Cfg::BTILE, b_full);
      pdl_wait();                             // weights are constants; activations must wait for the predecessor grids
      const uint64_t pol = l2_policy_stream();
      // mbarrier waits only see the phase parity, so a ring must have exactly one in-order consumer; tile i of this CTA
      // goes to ring i % nrings.
      int stage = 0, stage_other = 0;
      uint32_t phase = 0, phase_other = 0;   // (stage, phase) of the current tile's ring / of the other ring
      int it = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x, ++it) {
        const int n = tile / per_frame, rem = tile % per_frame;
        const int y0 = (rem / tiles_x) * 16, x0 = (rem % tiles_x) * 8;
        const int ring = nrings == 2 ? (it & 1) : 0, rbase = tc_ring_base(stages, ring), rsize = tc_ring_size(stages, ring);
        for (int c = 0; c < Cfg::KCH; ++c) {
          const int sidx = rbase + stage;
          mbar_wait(&empty[sidx], phase ^ 1);
          mbar_arrive_expect_tx(&full[sidx], Cfg::STAGE_PAYLOAD);
          uint8_t* dst = sA + (size_t)sidx * Cfg::STAGE_BYTES;
          if constexpr (Cfg::S2) {
#pragma unroll
            for (int i = 0; i < 4; ++i) {
              const int ph = i < 2 ? 1 : 0, pw = (i & 1) ? 0 : 1;
              tma_load_5d(dst + Cfg::SUB_OFF(i), &s2maps.m[i], &full[sidx], pw * p.in_C + p.in_c_off + c * Cfg::CW, x0 - pw, ph,
                          y0 - ph, n, pol);
            }
          } else {
            tma_load_4d(dst, &tmap, &full[sidx], c * Cfg::CW, x0 - Cfg::PAD, y0 - Cfg::PAD, n, pol);
          }
          if (++stage == rsize) { stage = 0; phase ^= 1; }
        }
        if (nrings == 2) { const int ts = stage; stage = stage_other; stage_other = ts; const uint32_t tp = phase; phase = phase_other; phase_other = tp; }
      }
    }
  } else if (warp >= 4 && (warp >> 2) <= nrings) {
    // ===================== consumers: warpgroup g takes the CTA's tiles g-1, g-1+nrings, ... =====================
    const int g = (warp >> 2) - 1, t = threadIdx.x & 127, wlane = threadIdx.x & 31;
    pdl_wait();                               // residual reads / output writes must follow the predecessor grids
    mbar_wait(b_full, 0);
    const uint32_t b_base = smem_u32(sB);
    const int rbase = tc_ring_base(stages, g), rsize = tc_ring_size(stages, g);
    int stage = 0;
    uint32_t phase = 0;
    for (int tile = blockIdx.x + g * gridDim.x; tile < num_tiles; tile += nrings * gridDim.x) {
      const int n = tile / per_frame, rem = tile % per_frame;
      const int y0 = (rem / tiles_x) * 16, x0 = (rem % tiles_x) * 8;
      float acc[2][NT / 2];   // SWAP: acc[0] .. acc[1] are the 64 registers of one m64n128 accumulator
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int j = 0; j < NT / 2; ++j) acc[h][j] = 0.f;
      uint32_t scale_d = 0;
      int prev = -1;
      for (int c = 0; c < Cfg::KCH; ++c) {
        const int sidx = rbase + stage;
        mbar_wait(&full[sidx], phase);
        uint8_t* a_stage = sA + (size_t)sidx * Cfg::STAGE_BYTES;
        if constexpr (EB == 4) {
          tf32_round_smem(a_stage, Cfg::STAGE_BYTES, t, 128);
          fence_proxy_async();                // generic-proxy writes -> visible to wgmma
          wg_bar_sync(1 + g);
        }
        const uint32_t a_base = smem_u32(a_stage);
        wgmma_fence();
#pragma unroll
        for (int tap = 0; tap < Cfg::TAPS; ++tap) {
          const int r = tap / Cfg::KS, s = tap % Cfg::KS;
          uint32_t a_tap, sbo;
          if constexpr (Cfg::S2) {
            const int sub = (r != 1 ? 0 : 2) + (s != 1 ? 0 : 1);
            const int bw = Cfg::BW(sub);
            a_tap = a_base + (uint32_t)(Cfg::SUB_OFF(sub) + ((r == 2 ? bw : 0) + (s == 2 ? 1 : 0)) * Cfg::ROWB);
            sbo = bw * Cfg::ROWB;
          } else {
            a_tap = a_base + (uint32_t)((r * Cfg::HW_ + s) * Cfg::ROWB);
            sbo = Cfg::HW_ * Cfg::ROWB;
          }
          const uint32_t b_tap = b_base + (uint32_t)((tap * Cfg::KCH + c) * Cfg::BTILE);
#pragma unroll
          for (int k = 0; k < Cfg::KSTEPS; ++k) {
            if (Cfg::FOLDABLE && !((kmask >> (tap * 2 + (k * 2) / Cfg::KSTEPS)) & 1u)) continue;
            const uint64_t bdesc = make_smem_desc(b_tap + k * 32, 8 * Cfg::ROWB, Cfg::LAYOUT);
            if constexpr (SWAP) {
              wgmma_n128_bf16(*reinterpret_cast<float(*)[64]>(&acc[0][0]), bdesc, make_smem_desc(a_tap + k * 32, sbo, Cfg::LAYOUT), scale_d);
            } else {
              wgmma_any<NT, EB>(acc[0], make_smem_desc(a_tap + k * 32, sbo, Cfg::LAYOUT), bdesc, scale_d);
              wgmma_any<NT, EB>(acc[1], make_smem_desc(a_tap + 8 * sbo + k * 32, sbo, Cfg::LAYOUT), bdesc, scale_d);
            }
            scale_d = 1;
          }
        }
        wgmma_commit();
        if (prev >= 0) {                      // the previous stage's MMAs have retired: hand it back to the producer
          wgmma_wait<1>();
          if (wlane == 0) mbar_arrive(&empty[prev]);
        }
        prev = sidx;
        if (++stage == rsize) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      if (wlane == 0) mbar_arrive(&empty[prev]);
      if constexpr (SWAP) {
        if (p.res != nullptr && p.res_dtype == B200ROMP_F32)
          wg_epilogue_swap<float2>(p, *reinterpret_cast<float(*)[64]>(&acc[0][0]), n, y0, x0, blockIdx.y * NT, t);
        else
          wg_epilogue_swap<uint32_t>(p, *reinterpret_cast<float(*)[64]>(&acc[0][0]), n, y0, x0, blockIdx.y * NT, t);
      } else {
        wg_epilogue<NT, GENERIC ? kEpiGeneric : kEpiNhwc>(p, acc, p.bias, n, y0, x0, blockIdx.y * NT, t);
      }
    }
  }
}

// Streamed weights as A (plan kind 34): bf16 3x3 stride 1, 256 input channels, 64-output-channel slabs, bf16 NHWC output.
// A 64-channel slab of 256 input channels (295 KB) does not fit next to a pipeline, so it streams through the stage ring
// with the input: stage = one 32-channel K chunk of the slab's 9 taps (36 KB, M = 64 rows of 64 B, the swizzled image of
// tc_pack_image) + the 18x18 halo of a 16x16 output tile (20 KB).  A work item is (tile, slab); both consumer warpgroups
// read every stage, warpgroup g taking the 8-column half g of the tile as B: N = 128, 16 8-pixel groups SBO = 18 halo rows
// apart, each tap a shifted descriptor.  Per k-step a warpgroup reads 2 + 4 KB for 128 pixels x 64 channels, where the
// N = 32 plan reads 2 x 3 KB for 128 x 32, and a frame's input is loaded 4 times (once per slab) instead of 8.  The slab
// costs 295 KB of L2 reads per item.  Chunks, taps and k-steps keep the order of conv_tc_kernel, so the fp32 sums are
// bit-identical.
constexpr int kStrmCin = 256, kStrmKch = kStrmCin / 32, kStrmRowB = 64, kStrmHalo = 18;
constexpr int kStrmWBytes = 9 * 64 * kStrmRowB;                                     // one K chunk of one slab
constexpr int kStrmHaloPayload = kStrmHalo * kStrmHalo * kStrmRowB;
constexpr int kStrmStageBytes = kStrmWBytes + (kStrmHaloPayload + 1023) / 1024 * 1024;
constexpr int kStrmStages = 3;
constexpr int kStrmSmem = kStrmStages * kStrmStageBytes + 1024 /*barriers*/ + 1024 /*align slack*/;
static_assert(kStrmSmem <= 227 * 1024, "streamed-weight stages do not fit shared memory");

__global__ void __launch_bounds__(kTcThreads, 1)
conv_tc_stream_kernel(const __grid_constant__ CUtensorMap tmap, const ConvParams p, const uint8_t* __restrict__ wpack, int tiles_x,
                      int tiles_y, int nslabs, int num_items) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + kStrmStages * kStrmStageBytes);
  uint64_t* empty = full + kStrmStages;
  const int warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) {
    for (int i = 0; i < kStrmStages; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], 8);   // one arrival per consumer warp: both warpgroups read every stage
    }
    fence_barrier_init();
  }
  __syncthreads();
  pdl_trigger();
  const int per_frame = tiles_x * tiles_y;

  if (warp == 0) {
    // ===================== producer: weights chunk + input halo per stage =====================
    if (elect_one()) {
      pdl_wait();
      const uint64_t pol = l2_policy_stream();
      int stage = 0;
      uint32_t phase = 0;
      for (int item = blockIdx.x; item < num_items; item += gridDim.x) {
        const int tile = item / nslabs, slab = item % nslabs;
        const int n = tile / per_frame, rem = tile % per_frame;
        const int y0 = (rem / tiles_x) * 16, x0 = (rem % tiles_x) * 16;
        for (int c = 0; c < kStrmKch; ++c) {
          mbar_wait(&empty[stage], phase ^ 1);
          mbar_arrive_expect_tx(&full[stage], kStrmWBytes + kStrmHaloPayload);
          uint8_t* dst = smem + (size_t)stage * kStrmStageBytes;
          bulk_copy_g2s(dst, wpack + ((size_t)slab * kStrmKch + c) * kStrmWBytes, kStrmWBytes, &full[stage]);
          tma_load_4d(dst + kStrmWBytes, &tmap, &full[stage], c * 32, x0 - 1, y0 - 1, n, pol);
          if (++stage == kStrmStages) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else if (warp >= 4) {
    // ===================== consumers: warpgroup g takes columns 8g .. 8g + 7 of every tile =====================
    const int g = (warp >> 2) - 1, t = threadIdx.x & 127, wlane = threadIdx.x & 31;
    pdl_wait();
    int stage = 0;
    uint32_t phase = 0;
    for (int item = blockIdx.x; item < num_items; item += gridDim.x) {
      const int tile = item / nslabs, slab = item % nslabs;
      const int n = tile / per_frame, rem = tile % per_frame;
      const int y0 = (rem / tiles_x) * 16, x0 = (rem % tiles_x) * 16;
      float acc[64];
#pragma unroll
      for (int j = 0; j < 64; ++j) acc[j] = 0.f;
      uint32_t scale_d = 0;
      int prev = -1;
      for (int c = 0; c < kStrmKch; ++c) {
        mbar_wait(&full[stage], phase);
        const uint32_t w_base = smem_u32(smem + (size_t)stage * kStrmStageBytes), a_base = w_base + kStrmWBytes;
        wgmma_fence();
#pragma unroll
        for (int tap = 0; tap < 9; ++tap) {
          const uint32_t a_tap = a_base + (uint32_t)(((tap / 3) * kStrmHalo + tap % 3 + 8 * g) * kStrmRowB);
#pragma unroll
          for (int k = 0; k < 2; ++k) {
            wgmma_n128_bf16(acc, make_smem_desc(w_base + tap * 64 * kStrmRowB + k * 32, 8 * kStrmRowB, kSw64),
                            make_smem_desc(a_tap + k * 32, kStrmHalo * kStrmRowB, kSw64), scale_d);
            scale_d = 1;
          }
        }
        wgmma_commit();
        if (prev >= 0) {                      // the previous stage's MMAs have retired: hand it back to the producer
          wgmma_wait<1>();
          if (wlane == 0) mbar_arrive(&empty[prev]);
        }
        prev = stage;
        if (++stage == kStrmStages) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      if (wlane == 0) mbar_arrive(&empty[prev]);
      if (p.res != nullptr && p.res_dtype == B200ROMP_F32) wg_epilogue_swap<float2>(p, acc, n, y0, x0 + 8 * g, slab * 64, t);
      else wg_epilogue_swap<uint32_t>(p, acc, n, y0, x0 + 8 * g, slab * 64, t);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
PFN_encodeTiled tc_get_encode() {
  static PFN_encodeTiled fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_encodeTiled>(ptr);
  });
  return fn;
}

int tc_encode_tiled(CUtensorMap* map, CUtensorMapDataType dtype, int rank, const void* base, const cuuint64_t* dims,
                    const cuuint64_t* strides, const cuuint32_t* box, CUtensorMapSwizzle swizzle, const char* tag) {
  PFN_encodeTiled encode = tc_get_encode();
  if (!encode) {
    set_error("%s: cuTensorMapEncodeTiled is unavailable", tag);
    return B200ROMP_ECUDA;
  }
  const cuuint32_t estr[5] = {1, 1, 1, 1, 1};
  const CUresult cr = encode(map, dtype, rank, const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                             swizzle, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (cr != CUDA_SUCCESS) {
    set_error("%s: cuTensorMapEncodeTiled failed with %d", tag, (int)cr);
    return B200ROMP_ECUDA;
  }
  return B200ROMP_OK;
}

int tc_encode_nhwc_input(CUtensorMap* map, const ConvParams& p, int eb, int box_c, int box_w, int box_h, CUtensorMapSwizzle swizzle,
                         const char* tag) {
  const cuuint64_t dims[4] = {(cuuint64_t)p.cin, (cuuint64_t)p.Win, (cuuint64_t)p.Hin, (cuuint64_t)p.B};
  const cuuint64_t strides[3] = {(cuuint64_t)p.in_C * eb, (cuuint64_t)p.Win * p.in_C * eb, (cuuint64_t)p.Hin * p.Win * p.in_C * eb};
  const cuuint32_t box[4] = {(cuuint32_t)box_c, (cuuint32_t)box_w, (cuuint32_t)box_h, 1};
  return tc_encode_tiled(map, eb == 2 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4,
                         static_cast<const uint8_t*>(p.in) + (size_t)p.in_c_off * eb, dims, strides, box, swizzle, tag);
}

float tc_round_tf32_host(float w) {
  uint32_t u;
  memcpy(&u, &w, 4);
  if ((u & 0x7F800000u) != 0x7F800000u) u = (u + 0x1000u) & ~0x1FFFu;
  float r;
  memcpy(&r, &u, 4);
  return r;
}

std::vector<uint8_t> tc_pack_image(const float* w_oihw, int cin, int cout, int taps, int nt, int rowb, int eb) {
  // shared-memory image [n-tile][tap][chunk][NT rows x rowb bytes] with the TMA/wgmma XOR swizzle; elements bf16 (eb = 2)
  // or fp32 rounded to TF32 (eb = 4)
  const int cw = rowb / eb, kch = cin / cw, ntiles = (cout + nt - 1) / nt, per16 = 16 / eb;
  std::vector<uint8_t> img((size_t)ntiles * taps * kch * nt * rowb, 0);
  for (int j = 0; j < ntiles; ++j)
    for (int t = 0; t < taps; ++t)
      for (int c = 0; c < kch; ++c) {
        uint8_t* tile = img.data() + (((size_t)j * taps + t) * kch + c) * nt * rowb;
        for (int n = 0; n < nt; ++n)
          for (int k = 0; k < cw; ++k) {
            const int co = j * nt + n, ci = c * cw + k;
            if (co >= cout) continue;                                     // zero rows pad cout up to a multiple of NT
            const float w = w_oihw[((size_t)co * cin + ci) * taps + t];
            const int chunk16 = k / per16;
            const int phase = rowb == 128 ? (n & 7) : ((n >> 1) & 3);     // Swizzle<3,4,3> / Swizzle<2,4,3>
            const size_t byte = (size_t)n * rowb + (size_t)((chunk16 ^ phase) * 16) + (k % per16) * eb;
            if (eb == 2) { const __nv_bfloat16 b = __float2bfloat16_rn(w); memcpy(tile + byte, &b, 2); }
            else { const float f = tc_round_tf32_host(w); memcpy(tile + byte, &f, 4); }
          }
      }
  return img;
}

int tc_pack_weights(const float* w_oihw, int cin, int cout, int taps, int nt, void** d_out, std::vector<void*>* allocs, int rowb, int eb) {
  const std::vector<uint8_t> img = tc_pack_image(w_oihw, cin, cout, taps, nt, rowb, eb);
  *d_out = upload(img.data(), img.size(), allocs);
  return *d_out ? B200ROMP_OK : B200ROMP_ECUDA;
}

std::string TcConvPlan::describe() const {
  char buf[128];
  snprintf(buf, sizeof(buf), " [tc%s k%d v%d nt%d grid %dx%d smem %d stages %d%s]%s", eb == 4 ? "-tf32" : "", kind / 10, kind % 10, nt,
           grid_x, grid_y, smem_bytes, stages, kmask != 0xFFFFFFFFu ? " pixel-pairs" : "", kind == 31 ? " [tc-swap weights-as-A n128]" : kind == 34 ? " [tc-stream weights-as-A n128 tile 16x16]" : "");
  return buf;
}

static bool tc_s2_supported(const ConvParams& p) {
  if ((p.in_dtype != B200ROMP_BF16 && p.in_dtype != B200ROMP_F32) || p.input_norm || p.out_nchw || p.pow_channel >= 0) return false;
  const int eb = p.in_dtype == B200ROMP_F32 ? 4 : 2;
  if (eb == 4 && (p.out_dtype != B200ROMP_F32 || (p.res != nullptr && p.res_dtype != B200ROMP_F32))) return false;
  if (p.cin != 32 && p.cin != 64 && p.cin != 128 && p.cin != 256) return false;
  if (eb == 4 && p.cin == 256) return false;                   // fp32 weights of 256 channels do not fit: the graph builder splits K
  if (p.in_C % 8 != 0 || p.in_c_off % 8 != 0) return false;    // channel slice [in_c_off, in_c_off + cin) of the merged (pw, c) dim
  if (p.cout % 32 != 0 || p.Hin % 2 != 0 || p.Win % 2 != 0) return false;
  if (p.Hout % 16 != 0 || p.Wout % 8 != 0 || p.Hout * 2 != p.Hin || p.Wout * 2 != p.Win) return false;
  if (p.out_C % 8 != 0 || p.out_c_off % 8 != 0) return false;
  if (p.res != nullptr && (p.res_C % 8 != 0 || p.res_c_off % 8 != 0)) return false;
  if ((reinterpret_cast<uintptr_t>(p.in) & 15) != 0) return false;
  return true;
}

static bool tc_shape_supported(const ConvParams& p, int ksize, int stride) {
  if (stride == 2 && ksize == 3) return tc_s2_supported(p);
  if (stride != 1 || (ksize != 1 && ksize != 3)) return false;
  if ((p.in_dtype != B200ROMP_BF16 && p.in_dtype != B200ROMP_F32) || p.input_norm) return false;   // F32 = the TF32 engine
  if (p.in_dtype == B200ROMP_F32 && (p.out_dtype != B200ROMP_F32 || (p.res != nullptr && p.res_dtype != B200ROMP_F32))) return false;
  if (p.cin != 32 && p.cin != 64 && p.cin != 128 && p.cin != 256) return false;
  if (p.Hout % 16 != 0 || p.Wout % 8 != 0) return false;
  if (p.in_C % 8 != 0 || p.in_c_off % 8 != 0) return false;             // TMA: 16 B aligned base and strides
  if (p.out_nchw) {                                                      // map outputs: any cout (padded to 32), scalar stores
    if (p.out_dtype != B200ROMP_F32 || p.up != 1 || p.res != nullptr) return false;
    return (reinterpret_cast<uintptr_t>(p.in) & 15) == 0;
  }
  if (p.pow_channel >= 0 || p.cout % 32 != 0) return false;
  if (p.out_C % 8 != 0 || p.out_c_off % 8 != 0) return false;           // vector epilogue
  if (p.res != nullptr && (p.res_C % 8 != 0 || p.res_c_off % 8 != 0)) return false;
  if ((reinterpret_cast<uintptr_t>(p.in) & 15) != 0) return false;
  return true;
}

static int tc_rowb(int ksize, int stride, int cin, int eb) { return stride == 2 ? s2_row_bytes(cin, eb) : tc_row_bytes(ksize, cin, eb); }

// the streamed-weight plan (kind 34, conv_tc_stream_kernel): bf16 3x3 stride 1, 256 -> 64k channels, 16x16 tiles, bf16 NHWC
// output at conv resolution
static bool tc_stream_eligible(const ConvParams& p, int ksize, int stride) {
  return ksize == 3 && stride == 1 && p.in_dtype == B200ROMP_BF16 && p.cin == kStrmCin && p.cout % 64 == 0 &&
         p.out_dtype == B200ROMP_BF16 && tc_nhwc_out(p, p.cout) && p.Hout % 16 == 0 && p.Wout % 16 == 0;
}

// kind, operand bytes, N tile, pipeline stages and shared memory of a plan: the weights stay resident next to >= 2 pipeline
// stages (>= 1 at stride 2).  false when they do not fit.
static bool tc_tile(const ConvParams& p, int ksize, int stride, TcConvPlan* plan) {
  const int eb = p.in_dtype == B200ROMP_F32 ? 4 : 2;
  const int rowb = tc_rowb(ksize, stride, p.cin, eb), kch = p.cin / (rowb / eb);
  const int budget = 227 * 1024 - 1024 /*align slack*/ - 1024 /*barriers*/;
  auto bbytes = [&](int n) { return ksize * ksize * kch * n * rowb; };
  if (tc_stream_eligible(p, ksize, stride)) {
    plan->kind = 34;
    plan->eb = 2;
    plan->cin = p.cin; plan->cout = p.cout; plan->nt = 64;
    plan->stages = kStrmStages;
    plan->smem_bytes = kStrmSmem;
    return true;
  }
  int nt = (p.cout % 64 == 0) ? 64 : 32;
  int stage_bytes, stages;
  if (stride == 2) {
    auto sub_bytes = [&](int i) { return ((i < 2 ? 17 : 16) * ((i & 1) ? 8 : 9) * rowb + 1023) / 1024 * 1024; };
    stage_bytes = sub_bytes(0) + sub_bytes(1) + sub_bytes(2) + sub_bytes(3);
    if (nt == 64 && bbytes(64) + 2 * stage_bytes > budget && bbytes(32) + 2 * stage_bytes <= budget) nt = 32;
    if (nt == 64 && bbytes(64) + stage_bytes > budget) nt = 32;
    if (bbytes(nt) + stage_bytes > budget) return false;
    stages = std::min(4, (budget - bbytes(nt)) / stage_bytes);
  } else {
    const int hh = 16 + 2 * (ksize / 2), hw = 8 + 2 * (ksize / 2);
    stage_bytes = (hh * hw * rowb + 1023) / 1024 * 1024;
    if (bbytes(nt) + 3 * stage_bytes > budget && nt == 64) nt = 32;
    if (bbytes(nt) + 2 * stage_bytes > budget && nt == 32) nt = 16;   // TF32 3x3 256 -> *: 288 KB of weights at N = 32
    if (bbytes(nt) + 2 * stage_bytes > budget) return false;
    stages = std::min((budget - bbytes(nt)) / stage_bytes, 8);   // split into two rings (one per consumer warpgroup)
  }
  plan->kind = stride == 2 ? 32 : ksize * 10;
  // the weights as A (SWAP): bf16 3x3 stride 1, 128 -> 128 channels at N = 64, bf16 NHWC output at conv resolution
  if (ksize == 3 && stride == 1 && eb == 2 && p.cin == 128 && p.cout == 128 && nt == 64 && p.out_dtype == B200ROMP_BF16 &&
      tc_nhwc_out(p, p.cout))
    plan->kind = 31;
  plan->eb = eb;
  plan->cin = p.cin; plan->cout = p.cout; plan->nt = nt;
  plan->stages = stages;
  plan->smem_bytes = bbytes(nt) + stages * stage_bytes + 1024 + 1024;
  return true;
}

bool tc_conv_supported(const ConvParams& p, int ksize, int stride) {
  TcConvPlan plan;
  return tc_shape_supported(p, ksize, stride) && tc_tile(p, ksize, stride, &plan);
}

template <int MODE, int CIN, int NT, int EB, bool SWAP = false>
static int launch_inst(const TcConvPlan& plan, const ConvParams& p, cudaStream_t stream, bool set_attr_only) {
  if (set_attr_only) {   // plans of one instantiation differ in stages
    if constexpr (SWAP) {
      B2R_CUDA_OK(cudaFuncSetAttribute(conv_tc_kernel<MODE, CIN, NT, EB, false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    } else {
      B2R_CUDA_OK(cudaFuncSetAttribute(conv_tc_kernel<MODE, CIN, NT, EB, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
      B2R_CUDA_OK(cudaFuncSetAttribute(conv_tc_kernel<MODE, CIN, NT, EB, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    }
    return B200ROMP_OK;
  }
  auto kern = SWAP ? conv_tc_kernel<MODE, CIN, NT, EB, false, SWAP>
                   : p.cout % NT == 0 && tc_nhwc_out(p, p.cout) ? conv_tc_kernel<MODE, CIN, NT, EB, false> : conv_tc_kernel<MODE, CIN, NT, EB, true>;
  const int tiles_x = p.Wout / 8, tiles_y = p.Hout / 16;
  const int num_tiles = tiles_x * tiles_y * p.B;
  dim3 grid(std::min(plan.grid_x, num_tiles), plan.grid_y);
  B2R_CUDA_OK(tc_launch(kern, grid, kTcThreads, plan.smem_bytes, stream, plan.tmap_in, plan.tmap_s2, p,
                        reinterpret_cast<const uint8_t*>(plan.d_wpack), tiles_x, tiles_y, num_tiles, plan.stages, plan.kmask));
  return B200ROMP_OK;
}

static int dispatch(const TcConvPlan& plan, const ConvParams& p, cudaStream_t stream, bool attr) {
  const int mode = plan.kind == 32 ? 2 : plan.kind / 10;
  if (plan.kind == 34) {
    if (attr) {
      B2R_CUDA_OK(cudaFuncSetAttribute(conv_tc_stream_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kStrmSmem));
      return B200ROMP_OK;
    }
    const int tiles_x = p.Wout / 16, tiles_y = p.Hout / 16, nslabs = p.cout / 64;
    const int num_items = tiles_x * tiles_y * p.B * nslabs;
    B2R_CUDA_OK(tc_launch(conv_tc_stream_kernel, dim3(std::min(plan.grid_x, num_items)), kTcThreads, plan.smem_bytes, stream, plan.tmap_in,
                          p, reinterpret_cast<const uint8_t*>(plan.d_wpack), tiles_x, tiles_y, nslabs, num_items));
    return B200ROMP_OK;
  }
  if (plan.kind == 31 && plan.cin == 128 && plan.nt == 64 && plan.eb == 2) return launch_inst<3, 128, 64, 2, true>(plan, p, stream, attr);
#define B2R_CASE(M, C, N, E) \
  if (mode == M && plan.cin == C && plan.nt == N && plan.eb == E) return launch_inst<M, C, N, E>(plan, p, stream, attr);
  // bf16
  B2R_CASE(3, 32, 32, 2) B2R_CASE(3, 32, 64, 2) B2R_CASE(3, 64, 32, 2) B2R_CASE(3, 64, 64, 2) B2R_CASE(3, 128, 32, 2) B2R_CASE(3, 128, 64, 2)
  B2R_CASE(3, 256, 32, 2) B2R_CASE(3, 256, 64, 2)
  B2R_CASE(1, 32, 32, 2) B2R_CASE(1, 32, 64, 2) B2R_CASE(1, 64, 32, 2) B2R_CASE(1, 64, 64, 2) B2R_CASE(1, 128, 32, 2) B2R_CASE(1, 128, 64, 2)
  B2R_CASE(1, 256, 32, 2) B2R_CASE(1, 256, 64, 2)
  B2R_CASE(2, 32, 32, 2) B2R_CASE(2, 32, 64, 2) B2R_CASE(2, 64, 32, 2) B2R_CASE(2, 64, 64, 2) B2R_CASE(2, 128, 32, 2) B2R_CASE(2, 256, 32, 2)
  // TF32 (fp32 tensors)
  B2R_CASE(3, 32, 32, 4) B2R_CASE(3, 32, 64, 4) B2R_CASE(3, 64, 32, 4) B2R_CASE(3, 64, 64, 4) B2R_CASE(3, 128, 32, 4) B2R_CASE(3, 256, 16, 4)
  B2R_CASE(1, 32, 32, 4) B2R_CASE(1, 32, 64, 4) B2R_CASE(1, 64, 32, 4) B2R_CASE(1, 64, 64, 4) B2R_CASE(1, 128, 32, 4) B2R_CASE(1, 128, 64, 4)
  B2R_CASE(1, 256, 32, 4) B2R_CASE(1, 256, 64, 4)
  B2R_CASE(2, 32, 32, 4) B2R_CASE(2, 32, 64, 4) B2R_CASE(2, 64, 32, 4) B2R_CASE(2, 128, 32, 4)
#undef B2R_CASE
  set_error("conv_tc: no instantiation for mode %d cin%d nt%d eb%d", mode, plan.cin, plan.nt, plan.eb);
  return B200ROMP_EINVAL;
}

int tc_conv_prepare(const ConvParams& p, int ksize, int stride, const float* w_oihw, int sm_count, TcConvPlan* plan,
                    std::vector<void*>* allocs) {
  if (!tc_tile(p, ksize, stride, plan)) {
    set_error("conv_tc: k%d s%d cin%d does not fit shared memory", ksize, stride, p.cin);
    return B200ROMP_EINVAL;
  }
  if (plan->kind == 34) {
    // the slab image [slab][tap][chunk][64 x 64 B] reordered to [slab][chunk][tap]: one stage's weights are contiguous
    const std::vector<uint8_t> img = tc_pack_image(w_oihw, p.cin, p.cout, 9, 64, kStrmRowB, 2);
    std::vector<uint8_t> strm(img.size());
    const size_t tile = 64 * kStrmRowB;
    for (int j = 0; j < p.cout / 64; ++j)
      for (int tap = 0; tap < 9; ++tap)
        for (int c = 0; c < kStrmKch; ++c)
          memcpy(strm.data() + (((size_t)j * kStrmKch + c) * 9 + tap) * tile, img.data() + (((size_t)j * 9 + tap) * kStrmKch + c) * tile, tile);
    plan->d_wpack = upload(strm.data(), strm.size(), allocs);
    if (!plan->d_wpack) return B200ROMP_ECUDA;
    plan->grid_x = sm_count;
    plan->grid_y = 1;
    const int rc = tc_encode_nhwc_input(&plan->tmap_in, p, 2, 32, kStrmHalo, kStrmHalo, CU_TENSOR_MAP_SWIZZLE_64B, "conv_tc (streamed)");
    if (rc) return rc;
    return dispatch(*plan, p, nullptr, true);
  }
  const int eb = plan->eb, rowb = tc_rowb(ksize, stride, p.cin, eb), cw = rowb / eb;
  plan->grid_y = (p.cout + plan->nt - 1) / plan->nt;
  plan->grid_x = std::max(1, sm_count / plan->grid_y);
  int rc = tc_pack_weights(w_oihw, p.cin, p.cout, ksize * ksize, plan->nt, &plan->d_wpack, allocs, rowb, eb);
  if (rc) return rc;
  const CUtensorMapSwizzle swizzle = rowb == 128 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B;
  if (stride == 2) {
    // one map per input parity over the space-to-depth view: dims ([pw*C+c], W/2, ph, H/2, N)
    const cuuint64_t C = (cuuint64_t)p.in_C;
    const cuuint64_t gdim[5] = {2 * C, (cuuint64_t)p.Win / 2, 2, (cuuint64_t)p.Hin / 2, (cuuint64_t)p.B};
    const cuuint64_t E = (cuuint64_t)eb;
    const cuuint64_t gstr[4] = {2 * C * E, (cuuint64_t)p.Win * C * E, 2 * (cuuint64_t)p.Win * C * E, (cuuint64_t)p.Hin * p.Win * C * E};
    const CUtensorMapDataType dtype = eb == 2 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32;
    for (int i = 0; i < 4; ++i) {
      const cuuint32_t box[5] = {(cuuint32_t)cw, (cuuint32_t)((i & 1) ? 8 : 9), 1, (cuuint32_t)(i < 2 ? 17 : 16), 1};
      rc = tc_encode_tiled(&plan->tmap_s2.m[i], dtype, 5, p.in, gdim, gstr, box, swizzle, "conv_tc (stride 2)");
      if (rc) return rc;
    }
  } else {
    const int hh = 16 + 2 * (ksize / 2), hw = 8 + 2 * (ksize / 2);
    rc = tc_encode_nhwc_input(&plan->tmap_in, p, eb, cw, hw, hh, swizzle, "conv_tc");
    if (rc) return rc;
  }
  return dispatch(*plan, p, nullptr, true);
}

int tc_conv_launch(const TcConvPlan& plan, const ConvParams& p, cudaStream_t stream) { return dispatch(plan, p, stream, false); }

}  // namespace b200romp
