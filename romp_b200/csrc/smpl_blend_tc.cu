// SMPL shape + pose blend on the tensor cores (lbs, simple_romp/romp/smpl.py:151-170):
//     v_posed[n, (v,c)] = v_template[(v,c)] + sum_k [betas | R[1:]-I](n, k) * [shapedirs ; posedirs](k, (v,c)),   K = 10 + 207
// = the (B*6890) x 207 contraction, as ONE wgmma GEMM  [persons x K'] x [K' x 20670]  per batch.
//
// Precision: the result feeds a 1e-4 tolerance on vertices of magnitude ~1; a single fp16 (or bf16) product leaves
// ~1e-4 (7e-4) max error, a two-term split ~6e-5 - not safe.  So both operands are split x = hi + lo (fp16 each, 22
// significant bits) and three products are accumulated in fp32:  hi*hi + lo*hi + hi*lo.  Each operand is stored and moved
// once: B' = [B_hi | B_lo] (448 halfs per vertex coordinate, built once at smpl_create), A' = [f_hi | f_lo] (448 halfs per
// person, written by smpl_pose_kernel).  A streamed B_hi chunk is multiplied by the resident f_hi AND f_lo chunks while it
// sits in shared memory, a B_lo chunk by f_hi.
//
// Kernel (one CTA = 128 persons x a slice of the 162 coordinate tiles of 128):
//   * warp 0 TMA-loads the CTA's 128 A' rows once (14 chunks of 32 halfs = 64 B rows, SWIZZLE_64B, 112 KB resident), then
//     streams B' per (coordinate tile, chunk) - 128 rows x 64 B - through a 6-stage mbarrier ring;
//   * warpgroups 1 and 2 each own 64 of the persons: per coordinate tile 10 wgmma m64n128k16 per B_hi chunk pair and B_lo
//     chunk, into 64 fp32 registers per thread; both consume every stage (empty barrier: 8 warp arrivals);
//   * epilogue from registers: + v_template, into the coordinate-tile-major v_posed buffer [81][capacity][256] that the
//     skinning kernel reads (smpl.cu).
#include "tc_device.cuh"

#include <algorithm>

namespace b200romp {

namespace {
constexpr int kBlK = 448;                 // B' / A': 2 x 224 (217 features zero-padded to 224): [hi | lo]
constexpr int kBlChunks = kBlK / 32;      // 14 chunks of 32 halfs = 64 B rows; chunk c < 7: hi, c >= 7: lo
constexpr int kBlCols = 20736;            // 20670 vertex coordinates padded to 81 x 256
constexpr int kBlN = 128;                 // coordinates per tile
constexpr int kBlColTiles = kBlCols / kBlN;
constexpr int kBlChunkBytes = 128 * 64;   // 128 rows x 64 B (A': persons, B': coordinates)
constexpr int kBlABytes = kBlChunks * kBlChunkBytes;    // 114,688
constexpr int kBlStages = 6;
constexpr int kBlThreads = 384;           // warp 0 producer, warpgroups 1-2 consumers
constexpr int kBlendSmem = kBlABytes + kBlStages * kBlChunkBytes + 256 + 1024;

__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
               ::"r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1) : "memory");
}

#define B2R_BL_R8(i) "+f"(d[i + 0]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3]), "+f"(d[i + 4]), "+f"(d[i + 5]), "+f"(d[i + 6]), "+f"(d[i + 7])
__device__ __forceinline__ void wgmma_f16_n128(float (&d)[64], uint64_t a, uint64_t b, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, "
      "%40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "%64, %65, p, 1, 1, 0, 0;\n\t}"
      : B2R_BL_R8(0), B2R_BL_R8(8), B2R_BL_R8(16), B2R_BL_R8(24), B2R_BL_R8(32), B2R_BL_R8(40), B2R_BL_R8(48), B2R_BL_R8(56)
      : "l"(a), "l"(b), "r"(scale_d)
      : "memory");
}
#undef B2R_BL_R8

struct BlendMaps {
  CUtensorMap a, b;
};
}  // namespace

__global__ void __launch_bounds__(kBlThreads, 1)
smpl_blend_tc_kernel(const __grid_constant__ BlendMaps maps, const float* __restrict__ v_template /*[20736], zero padded*/, int n_host,
                     const int* __restrict__ d_count, int col_splits, float* __restrict__ v_posed /*[81][cap][256]*/, int cap) {
  const int count = d_count ? min(*d_count, n_host) : n_host;
  const int p0 = (blockIdx.x / col_splits) * 128, split = blockIdx.x % col_splits;
  if (p0 >= count) return;                    // whole CTA, before any barrier exists
  const int ct0 = split * kBlColTiles / col_splits, ct1 = (split + 1) * kBlColTiles / col_splits;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* sA = smem;                                  // 14 x [128 persons x 64 B]
  uint8_t* sB = sA + kBlABytes;                        // kBlStages x [128 coordinates x 64 B]
  uint64_t* full = reinterpret_cast<uint64_t*>(sB + kBlStages * kBlChunkBytes);
  uint64_t* empty = full + kBlStages;
  uint64_t* a_full = empty + kBlStages;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    for (int i = 0; i < kBlStages; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], 8);                // every warp of both consumer warpgroups
    }
    mbar_init(a_full, 1);
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == 0) {
    if (elect_one()) {
      mbar_arrive_expect_tx(a_full, kBlABytes);
      for (int c = 0; c < kBlChunks; ++c) tma_load_2d(sA + c * kBlChunkBytes, &maps.a, a_full, c * 32, p0);
      int stage = 0;
      uint32_t phase = 0;
      for (int ct = ct0; ct < ct1; ++ct) {
        for (int c = 0; c < kBlChunks; ++c) {
          mbar_wait(&empty[stage], phase ^ 1);
          mbar_arrive_expect_tx(&full[stage], kBlChunkBytes);
          tma_load_2d(sB + stage * kBlChunkBytes, &maps.b, &full[stage], c * 32, ct * kBlN);
          if (++stage == kBlStages) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else if (warp >= 4) {
    const int g = (warp >> 2) - 1, w = warp & 3;
    const uint32_t a_base = smem_u32(sA) + g * 64 * 64;   // this warpgroup's 64 persons of every A' chunk
    mbar_wait(a_full, 0);
    int stage = 0;
    uint32_t phase = 0;
    for (int ct = ct0; ct < ct1; ++ct) {
      float acc[64];
      uint32_t scale_d = 0;
      int prev = -1;
#pragma unroll
      for (int c = 0; c < kBlChunks; ++c) {
        mbar_wait(&full[stage], phase);
        const uint32_t b_base = smem_u32(sB + stage * kBlChunkBytes);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 2; ++k) {
          const uint64_t bdesc = make_smem_desc(b_base + k * 32, 8 * 64, kSw64);
          // B_hi chunk c: f_hi (A' chunk c) and f_lo (A' chunk 7 + c);  B_lo chunk c: f_hi (A' chunk c - 7)
          const int a0 = c < 7 ? c : c - 7;
          wgmma_f16_n128(acc, make_smem_desc(a_base + a0 * kBlChunkBytes + k * 32, 8 * 64, kSw64), bdesc, scale_d);
          scale_d = 1;
          if (c < 7) wgmma_f16_n128(acc, make_smem_desc(a_base + (7 + c) * kBlChunkBytes + k * 32, 8 * 64, kSw64), bdesc, 1);
        }
        wgmma_commit();
        if (prev >= 0) {                      // the previous stage's MMAs have retired: hand it back to the producer
          wgmma_wait<1>();
          if (lane == 0) mbar_arrive(&empty[prev]);
        }
        prev = stage;
        if (++stage == kBlStages) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      if (lane == 0) mbar_arrive(&empty[prev]);
      // accumulator fragment: thread (w, lane) holds columns 8j + 2(lane%4) + {0,1} of rows 16w + lane/4 (+8)
      float* vp = v_posed + ((size_t)(ct >> 1) * cap) * 256 + (ct & 1) * kBlN;
#pragma unroll
      for (int j = 0; j < kBlN / 8; ++j) {
        const int col = 8 * j + 2 * (lane & 3);
        const float2 vt = *reinterpret_cast<const float2*>(v_template + ct * kBlN + col);
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int p = p0 + 64 * g + 16 * w + (lane >> 2) + 8 * e;
          if (p < count)
            *reinterpret_cast<float2*>(vp + (size_t)p * 256 + col) = make_float2(acc[4 * j + 2 * e] + vt.x, acc[4 * j + 2 * e + 1] + vt.y);
        }
      }
    }
  }
}

// a_rows: fp16 [cap] rows of 448 inside the per-person scratch records of smpl.cu (`row_stride_bytes` apart);  v_posed: fp32
// [81][capacity][256], coordinate-tile major
int smpl_blend_tc_launch(const void* a_rows, int row_stride_bytes, int capacity, const void* b_rows /*fp16 [20736][448]*/,
                         float* v_posed, const float* v_template_pad, int n, const int* d_count, int sm_count, cudaStream_t stream) {
  BlendMaps m;
  const cuuint32_t box[2] = {32, 128};
  const cuuint64_t a_dim[2] = {(cuuint64_t)kBlK, (cuuint64_t)capacity}, a_str[1] = {(cuuint64_t)row_stride_bytes};
  const cuuint64_t b_dim[2] = {(cuuint64_t)kBlK, (cuuint64_t)kBlCols}, b_str[1] = {(cuuint64_t)kBlK * 2};
  const CUtensorMapDataType f16 = CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
  int rc = tc_encode_tiled(&m.a, f16, 2, a_rows, a_dim, a_str, box, CU_TENSOR_MAP_SWIZZLE_64B, "smpl_blend_tc (A')");
  if (!rc) rc = tc_encode_tiled(&m.b, f16, 2, b_rows, b_dim, b_str, box, CU_TENSOR_MAP_SWIZZLE_64B, "smpl_blend_tc (B')");
  if (rc) return rc;
  static bool attr_set = false;
  if (!attr_set) {
    B2R_CUDA_OK(cudaFuncSetAttribute(smpl_blend_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kBlendSmem));
    attr_set = true;
  }
  // `n` is the host-side upper bound of the person count (the device count may be smaller: surplus CTAs exit at once).
  // Few person tiles: split the coordinate tiles over more CTAs so that every SM has work.
  const int ptiles = (n + 127) / 128;
  const int col_splits = std::max(1, std::min(kBlColTiles, sm_count / std::max(1, ptiles)));
  smpl_blend_tc_kernel<<<ptiles * col_splits, kBlThreads, kBlendSmem, stream>>>(m, v_template_pad, n, d_count, col_splits, v_posed, capacity);
  B2R_CUDA_OK(cudaGetLastError());
  return B200ROMP_OK;
}

}  // namespace b200romp
