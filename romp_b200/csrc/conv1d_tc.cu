// wgmma GEMM for BEV's bird's-eye-view Conv1d stack (simple_romp/bev/model.py:24-45,179-182: three BasicBlock_1D =
// six Conv1d(k=3, pad=1)+BN1d+ReLU, 2560 -> 512 -> 512 | 512 -> 512 | 512 -> 128 -> 128, over the 128 image columns).
//
// The activation is the NHWC "image" [B, 1, W = 128, C] (channels innermost = K-major rows), ksize code 13 = 1x3.
//   GEMM M = 128 positions (one row of one frame; two wgmma m64 halves), N = NT output channels, K = 3 taps x Cin.
//   A: one TMA load per (tile, 64-channel chunk) of the 130-position halo row (x0 = -1, out-of-bounds = zero padding);
//      the 3 taps are 3 shared-memory descriptors shifted by one 128 B row each (same trick as conv_tc.cu).
//   B: Cin = 2560 makes the weights of one N tile 983 KB - not resident: each pipeline stage carries its own
//      [3 taps][NT rows x 128 B] weight slab (24 KB for NT = 64) next to the A row (17 KB); weights are packed
//      chunk-major so the slab of a stage is one contiguous bulk copy.
//   D: fp32 in registers of the consumer warpgroup; register epilogue: + bias, (+ residual), ReLU, dtype.
// Warps: 0 = TMA producer, 4-7 = consumer warpgroup (wgmma + epilogue).
#include "conv_tc.cuh"
#include "tc_device.cuh"

namespace b200romp {

constexpr int k1dThreads = 256;
constexpr int k1dARows = 130;
constexpr int k1dABytes = (k1dARows * 128 + 1023) / 1024 * 1024;   // 17408

template <int NT>
struct C1dCfg {
  static constexpr int BBYTES = 3 * NT * 128;
  static constexpr int STAGE_BYTES = k1dABytes + BBYTES;
};

template <int NT>
__global__ void __launch_bounds__(k1dThreads, 1)
conv1d_tc_kernel(const __grid_constant__ CUtensorMap tmap, const ConvParams p, const uint8_t* __restrict__ wpack, int kch, int tiles_w,
                 int num_tiles, int stages) {
  using Cfg = C1dCfg<NT>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + (size_t)stages * Cfg::STAGE_BYTES);
  uint64_t* empty = full + stages;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    for (int i = 0; i < stages; ++i) { mbar_init(&full[i], 1); mbar_init(&empty[i], 4); }
    fence_barrier_init();
  }
  __syncthreads();
  pdl_trigger();

  if (warp == 0) {
    if (elect_one()) {
      pdl_wait();
      const uint64_t pol = l2_policy_stream();
      int stage = 0;
      uint32_t phase = 0;
      const uint8_t* wsrc = wpack + (size_t)blockIdx.y * kch * Cfg::BBYTES;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int row = tile / tiles_w, x0 = (tile % tiles_w) * 128;
        for (int c = 0; c < kch; ++c) {
          mbar_wait(&empty[stage], phase ^ 1);
          uint8_t* dst = smem + (size_t)stage * Cfg::STAGE_BYTES;
          mbar_arrive_expect_tx(&full[stage], k1dARows * 128 + Cfg::BBYTES);
          tma_load_3d(dst, &tmap, &full[stage], p.in_c_off + c * 64, x0 - 1, row, pol);
          bulk_copy_g2s(dst + k1dABytes, wsrc + (size_t)c * Cfg::BBYTES, Cfg::BBYTES, &full[stage]);
          if (++stage == stages) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else if (warp >= 4) {
    const int t = threadIdx.x & 127;
    pdl_wait();
    int stage = 0;
    uint32_t phase = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      const int row = tile / tiles_w, x0 = (tile % tiles_w) * 128;
      float acc[2][NT / 2];
      uint32_t scale_d = 0;
      int prev = -1;
      for (int c = 0; c < kch; ++c) {
        mbar_wait(&full[stage], phase);
        const uint32_t a_base = smem_u32(smem + (size_t)stage * Cfg::STAGE_BYTES);
        const uint32_t b_base = a_base + k1dABytes;
        wgmma_fence();
#pragma unroll
        for (int tap = 0; tap < 3; ++tap) {
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            const uint64_t bdesc = make_smem_desc(b_base + tap * NT * 128 + k * 32, 1024, kSw128);
            wgmma_any<NT, 2>(acc[0], make_smem_desc(a_base + tap * 128 + k * 32, 1024, kSw128), bdesc, scale_d);
            wgmma_any<NT, 2>(acc[1], make_smem_desc(a_base + (64 + tap) * 128 + k * 32, 1024, kSw128), bdesc, scale_d);
            scale_d = 1;
          }
        }
        wgmma_commit();
        if (prev >= 0) {                      // the previous stage's MMAs have retired: hand it back to the producer
          wgmma_wait<1>();
          if (lane == 0) mbar_arrive(&empty[prev]);
        }
        prev = stage;
        if (++stage == stages) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      if (lane == 0) mbar_arrive(&empty[prev]);
      wg_epilogue<NT>(p, acc, p.bias, 0, row, x0, blockIdx.y * NT, t, /*linear=*/true);
    }
  }
}

// ------------------------------------------------------------------------------------------------
bool tc_conv1d_supported(const ConvParams& p) {
  if (p.in_dtype != B200ROMP_BF16 || p.input_norm || p.out_nchw || p.pow_channel >= 0 || p.up != 1) return false;
  if (p.cin % 64 != 0 || p.cout % 32 != 0 || p.Wout % 128 != 0 || p.Wout != p.Win || p.Hout != p.Hin) return false;
  if (p.in_C % 8 != 0 || p.in_c_off % 8 != 0 || p.out_C % 8 != 0 || p.out_c_off % 8 != 0) return false;
  if (p.res != nullptr && (p.res_C % 8 != 0 || p.res_c_off % 8 != 0 || p.res_broadcast)) return false;
  return true;
}

static int conv1d_encode(const ConvParams& p, TcConvPlan* plan) {
  const cuuint64_t gdim[3] = {(cuuint64_t)p.in_C, (cuuint64_t)p.Win, (cuuint64_t)p.B * p.Hin};
  const cuuint64_t gstr[2] = {(cuuint64_t)p.in_C * 2, (cuuint64_t)p.Win * p.in_C * 2};
  const cuuint32_t box[3] = {64, (cuuint32_t)k1dARows, 1};
  int rc = tc_encode_tiled(&plan->tmap_in, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 3, p.in, gdim, gstr, box, CU_TENSOR_MAP_SWIZZLE_128B,
                           "conv1d_tc");
  if (rc) return rc;
  plan->encoded_in = p.in;
  plan->encoded_batch = p.B;
  return B200ROMP_OK;
}

template <int NT>
static int conv1d_inst(const TcConvPlan& plan, const ConvParams& p, cudaStream_t stream, bool attr) {
  auto kern = conv1d_tc_kernel<NT>;
  if (attr) {
    B2R_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    return B200ROMP_OK;
  }
  const int tiles_w = p.Wout / 128, num_tiles = tiles_w * p.Hout * p.B;
  dim3 grid(std::min(plan.grid_x, num_tiles), plan.grid_y);
  B2R_CUDA_OK(tc_launch(kern, grid, k1dThreads, plan.smem_bytes, stream, plan.tmap_in, p, reinterpret_cast<const uint8_t*>(plan.d_wpack),
                        plan.cin / 64, tiles_w, num_tiles, plan.stages));
  return B200ROMP_OK;
}

int tc_conv1d_prepare(const ConvParams& p, const float* w_oi3, int sm_count, TcConvPlan* plan, std::vector<void*>* allocs) {
  const int nt = (p.cout % 64 == 0) ? 64 : 32;
  const int kch = p.cin / 64, ntiles = p.cout / nt;
  const int stage_bytes = k1dABytes + 3 * nt * 128;
  plan->kind = 13; plan->eb = 2;
  plan->cin = p.cin; plan->cout = p.cout; plan->nt = nt;
  plan->stages = std::min(6, (227 * 1024 - 2048) / stage_bytes);
  plan->grid_y = ntiles;
  plan->grid_x = std::max(1, sm_count / ntiles);
  plan->smem_bytes = plan->stages * stage_bytes + 2048;
  // weights: [ntile][chunk][tap][nt rows x 128 B], SWIZZLE_128B inside each (tap) tile; w_oi3 = [cout][cin][3]
  std::vector<__nv_bfloat16> img((size_t)ntiles * kch * 3 * nt * 64, __float2bfloat16_rn(0.f));
  for (int j = 0; j < ntiles; ++j)
    for (int c = 0; c < kch; ++c)
      for (int t = 0; t < 3; ++t) {
        __nv_bfloat16* tile = img.data() + ((((size_t)j * kch + c) * 3 + t) * nt) * 64;
        for (int n = 0; n < nt; ++n)
          for (int k = 0; k < 64; ++k) {
            const float w = w_oi3[((size_t)(j * nt + n) * p.cin + c * 64 + k) * 3 + t];
            const size_t byte = (size_t)n * 128 + (size_t)(((k / 8) ^ (n & 7)) * 16) + (k % 8) * 2;
            tile[byte / 2] = __float2bfloat16_rn(w);
          }
      }
  plan->d_wpack = upload(img.data(), img.size() * sizeof(__nv_bfloat16), allocs);
  if (!plan->d_wpack) return B200ROMP_ECUDA;
  if (!tc_get_encode()) {   // resolved now rather than at the first launch, which may be inside a stream capture
    set_error("conv1d_tc: cuTensorMapEncodeTiled is unavailable");
    return B200ROMP_ECUDA;
  }
  return nt == 64 ? conv1d_inst<64>(*plan, p, nullptr, true) : conv1d_inst<32>(*plan, p, nullptr, true);
}

// the input of the bird's-eye graph is an EXTERNAL tensor (assembled by b200romp_bev_bv_input): the tensor map is encoded
// at the first launch and again whenever the bound pointer (or the batch) differs from the one it was built for
int tc_conv1d_launch(TcConvPlan& plan, const ConvParams& p, cudaStream_t stream) {
  if (plan.encoded_in != p.in || plan.encoded_batch != p.B) {
    int rc = conv1d_encode(p, &plan);
    if (rc) return rc;
  }
  return plan.nt == 64 ? conv1d_inst<64>(plan, p, stream, false) : conv1d_inst<32>(plan, p, stream, false);
}

}  // namespace b200romp
