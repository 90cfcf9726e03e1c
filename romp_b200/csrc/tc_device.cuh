// Device-side building blocks shared by the tensor-core kernels (conv_tc.cu, conv_stem_tc.cu, conv1d_tc.cu): PTX wrappers
// for mbarrier / TMA / wgmma, the shared-memory matrix descriptor, and the register-accumulator epilogue.
#pragma once
#include <cuda.h>

#include <vector>

#include "conv_tc.cuh"

namespace b200romp {

// ------------------------------------------------------------------------------------------------
// PTX wrappers
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.b32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded wait: a protocol bug must not hang the GPU - trap after ~2 s instead.  (No printf here: a function call inside
// the consumer loop makes ptxas serialize every wgmma of the kernel.)
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  while (!mbar_try_wait(bar, parity)) {
    if (clock64() - t0 > 4000000000LL) __trap();
  }
}
__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile("{\n\t.reg .pred p;\n\telect.sync _|p, 0xffffffff;\n\tselp.b32 %0, 1, 0, p;\n\t}" : "=r"(pred));
  return pred != 0;
}
// Programmatic dependent launch: the next conv of the stream may start its prologue (barrier init, weight-slab copy - all
// independent of activations) while this grid drains; pdl_wait() then blocks until every predecessor grid has completed and
// its writes are visible.  Both are no-ops for a launch without the attribute.
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// barrier over the 128 threads of one warpgroup (ids 1.. ; 0 is __syncthreads)
__device__ __forceinline__ void wg_bar_sync(int id) { asm volatile("bar.sync %0, 128;" ::"r"(id) : "memory"); }

__device__ __forceinline__ uint64_t l2_policy_stream() {
  uint64_t pol;
  asm volatile("createpolicy.fractional.L2::evict_normal.b64 %0, 1.0;" : "=l"(pol));
  return pol;
}
__device__ __forceinline__ void tma_load_3d(void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2, uint64_t pol) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1, {%3, %4, %5}], [%2], %6;"
      ::"r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "l"(pol)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2, int c3, uint64_t pol) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1, {%3, %4, %5, %6}], [%2], %7;"
      ::"r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "l"(pol)
      : "memory");
}
__device__ __forceinline__ void tma_load_5d(void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1, int c2, int c3,
                                            int c4, uint64_t pol) {
  asm volatile(
      "cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1, {%3, %4, %5, %6, %7}], [%2], %8;"
      ::"r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4), "l"(pol)
      : "memory");
}
__device__ __forceinline__ void bulk_copy_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}

// ---- wgmma (sm_90a): D[64 x N] (+)= A[64 x K] * B[N x K]^T, both operands K-major in shared memory, fp32 accumulators in
// registers of the issuing warpgroup.  EB = 2: bf16 operands (K = 16 per instruction); EB = 4: fp32 storage consumed as TF32
// (K = 8).  Either way one instruction consumes 32 bytes of every operand row, so the shared-memory geometry of the kernels
// is expressed in BYTES and the TF32 engine is the same pipeline with twice the bytes per channel.
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

#define B2R_WG_R8(i) "+f"(d[i + 0]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3]), "+f"(d[i + 4]), "+f"(d[i + 5]), "+f"(d[i + 6]), "+f"(d[i + 7])
__device__ __forceinline__ void wgmma_n16(float (&d)[8], uint64_t a, uint64_t b, uint32_t scale_d, bool tf32) {
  if (!tf32)
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1, 0, 0;\n\t}"
        : B2R_WG_R8(0)
        : "l"(a), "l"(b), "r"(scale_d)
        : "memory");
  else
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n16k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1;\n\t}"
        : B2R_WG_R8(0)
        : "l"(a), "l"(b), "r"(scale_d)
        : "memory");
}
__device__ __forceinline__ void wgmma_n32(float (&d)[16], uint64_t a, uint64_t b, uint32_t scale_d, bool tf32) {
  if (!tf32)
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, "
        "%16, %17, p, 1, 1, 0, 0;\n\t}"
        : B2R_WG_R8(0), B2R_WG_R8(8)
        : "l"(a), "l"(b), "r"(scale_d)
        : "memory");
  else
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, "
        "%16, %17, p, 1, 1;\n\t}"
        : B2R_WG_R8(0), B2R_WG_R8(8)
        : "l"(a), "l"(b), "r"(scale_d)
        : "memory");
}
__device__ __forceinline__ void wgmma_n64(float (&d)[32], uint64_t a, uint64_t b, uint32_t scale_d, bool tf32) {
  if (!tf32)
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, "
        "%15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n\t}"
        : B2R_WG_R8(0), B2R_WG_R8(8), B2R_WG_R8(16), B2R_WG_R8(24)
        : "l"(a), "l"(b), "r"(scale_d)
        : "memory");
  else
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, "
        "%15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1;\n\t}"
        : B2R_WG_R8(0), B2R_WG_R8(8), B2R_WG_R8(16), B2R_WG_R8(24)
        : "l"(a), "l"(b), "r"(scale_d)
        : "memory");
}
// bf16 only: the N = 256 conv3 of the fused Bottleneck (conv_bottleneck_tc.cu) runs as two of these per warpgroup
__device__ __forceinline__ void wgmma_n128_bf16(float (&d)[64], uint64_t a, uint64_t b, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, "
      "%15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, "
      "%39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, "
      "%63}, %64, %65, p, 1, 1, 0, 0;\n\t}"
      : B2R_WG_R8(0), B2R_WG_R8(8), B2R_WG_R8(16), B2R_WG_R8(24), B2R_WG_R8(32), B2R_WG_R8(40), B2R_WG_R8(48), B2R_WG_R8(56)
      : "l"(a), "l"(b), "r"(scale_d)
      : "memory");
}
// bf16 only: conv1 of the folded BasicBlock (conv_block_tc.cu), 192 mid pixels per warpgroup
__device__ __forceinline__ void wgmma_n192_bf16(float (&d)[96], uint64_t a, uint64_t b, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %98, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n192k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, "
      "%15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, "
      "%39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, "
      "%63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, "
      "%87, %88, %89, %90, %91, %92, %93, %94, %95}, %96, %97, p, 1, 1, 0, 0;\n\t}"
      : B2R_WG_R8(0), B2R_WG_R8(8), B2R_WG_R8(16), B2R_WG_R8(24), B2R_WG_R8(32), B2R_WG_R8(40), B2R_WG_R8(48), B2R_WG_R8(56),
        B2R_WG_R8(64), B2R_WG_R8(72), B2R_WG_R8(80), B2R_WG_R8(88)
      : "l"(a), "l"(b), "r"(scale_d)
      : "memory");
}
#undef B2R_WG_R8
template <int NT, int EB>
__device__ __forceinline__ void wgmma_any(float (&d)[NT / 2], uint64_t a, uint64_t b, uint32_t scale_d) {
  if constexpr (NT == 64) wgmma_n64(d, a, b, scale_d, EB == 4);
  else if constexpr (NT == 32) wgmma_n32(d, a, b, scale_d, EB == 4);
  else wgmma_n16(d, a, b, scale_d, EB == 4);
}

// Shared-memory matrix descriptor of wgmma, K-major, swizzled:
//   [0,14) start>>4 | [16,30) LBO>>4 (=1, unused for swizzled K-major) | [32,46) SBO>>4 = byte distance between 8-row groups |
//   [49,52) base offset = 0 (pattern anchored at 1024 B) | [62,64) layout: 1 = SWIZZLE_128B, 2 = SWIZZLE_64B
constexpr uint32_t kSw128 = 1, kSw64 = 2;
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t addr, uint32_t sbo_bytes, uint32_t layout) {
  return (uint64_t)((addr & 0x3FFFF) >> 4) | ((uint64_t)1 << 16) | ((uint64_t)(sbo_bytes >> 4) << 32) | ((uint64_t)layout << 62);
}
__host__ __device__ constexpr uint32_t tc_layout(int row_bytes) { return row_bytes == 128 ? kSw128 : kSw64; }

// bytes of one shared-memory pixel row (= swizzle span) of a conv's A / B tiles.  The weight-heavy 3x3 layers
// (Cin >= 128) use half rows: more, smaller pipeline stages next to the resident weight slab.
__host__ __device__ constexpr int tc_row_bytes(int ksize, int cin, int eb) {
  return (ksize == 3 && cin >= 128) ? 64 : (cin * eb < 128 ? cin * eb : 128);
}

// ---- TF32 rounding of landed A tiles (EB = 4 kernels) -------------------------------------------------
// wgmma .tf32 reads fp32 containers and ignores the low 13 mantissa bits (truncation).  Truncating the activations of the
// ~100-layer stack biases the maps, so the TF32 engine does what a cvt.rna.tf32.f32 in front of mma.sync does
// in cuDNN/cuBLAS TF32 kernels: the consumer warpgroup rounds every landed A tile in place (shared memory, ties away from
// zero) before its MMAs.  Tensors in HBM stay exact fp32.
__device__ __forceinline__ uint32_t tf32_rna(uint32_t x) {
  uint32_t y;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(y) : "r"(x));
  return y;
}
__device__ __forceinline__ void tf32_round_smem(uint8_t* base, int bytes, int t, int nthreads) {
  const uint32_t s0 = smem_u32(base);
  for (int off = t * 16; off < bytes; off += nthreads * 16) {
    uint32_t a, b, c, d;
    asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(a), "=r"(b), "=r"(c), "=r"(d) : "r"(s0 + off));
    a = tf32_rna(a); b = tf32_rna(b); c = tf32_rna(c); d = tf32_rna(d);
    asm volatile("st.shared.v4.b32 [%4], {%0, %1, %2, %3};" ::"r"(a), "r"(b), "r"(c), "r"(d), "r"(s0 + off) : "memory");
  }
}

// ---- register epilogue --------------------------------------------------------------------------------
// Two consecutive output channels [co, co+1) of conv-output pixel (n, oy, ox), bias already added: residual, ReLU,
// nearest-upsample replication and dtype conversion with 8 / 4 byte accesses; NCHW maps, 1.1**x and partial channel
// tiles go through the generic scalar epilogue.
__device__ __forceinline__ void wg_store2(const ConvParams& p, int n, int oy, int ox, int co, float v0, float v1) {
  if (p.out_nchw || p.pow_channel >= 0 || co + 2 > p.cout) {
    const float v[2] = {v0, v1};
    conv_epilogue_store<2>(p, n, oy, ox, co, v);
    return;
  }
  const int up = p.up, Hf = p.Hout * up, Wf = p.Wout * up;
  for (int dy = 0; dy < up; ++dy) {
    for (int dx = 0; dx < up; ++dx) {
      const int fy = oy * up + dy, fx = ox * up + dx;
      const size_t pix = ((size_t)n * Hf + fy) * Wf + fx;
      float a = v0, b = v1;
      if (p.res != nullptr) {
        const size_t ri = ((size_t)(p.res_broadcast ? 0 : n) * Hf + fy) * Wf + fx;
        const size_t idx = ri * p.res_C + p.res_c_off + co;
        if (p.res_dtype == B200ROMP_BF16) {
          const __nv_bfloat162 r = *reinterpret_cast<const __nv_bfloat162*>(reinterpret_cast<const __nv_bfloat16*>(p.res) + idx);
          a += __low2float(r); b += __high2float(r);
        } else {
          const float2 r = *reinterpret_cast<const float2*>(reinterpret_cast<const float*>(p.res) + idx);
          a += r.x; b += r.y;
        }
      }
      if (p.relu) { a = fmaxf(a, 0.f); b = fmaxf(b, 0.f); }
      const size_t oi = pix * p.out_C + p.out_c_off + co;
      if (p.out_dtype == B200ROMP_BF16)
        *reinterpret_cast<__nv_bfloat162*>(reinterpret_cast<__nv_bfloat16*>(p.out) + oi) = __floats2bfloat162_rn(a, b);
      else
        *reinterpret_cast<float2*>(reinterpret_cast<float*>(p.out) + oi) = make_float2(a, b);
    }
  }
}

// output NHWC at conv resolution, channels [.., co_end) inside the op's channels: no NCHW maps, 1.1**x or upsampling
__host__ __device__ __forceinline__ bool tc_nhwc_out(const ConvParams& p, int co_end) {
  return p.up == 1 && !p.out_nchw && p.pow_channel < 0 && co_end <= p.cout;
}

__device__ __forceinline__ float2 res_pair(uint32_t r) {
  const __nv_bfloat162 v = *reinterpret_cast<const __nv_bfloat162*>(&r);
  return make_float2(__low2float(v), __high2float(v));
}
__device__ __forceinline__ float2 res_pair(float2 r) { return r; }

// NHWC output at conv resolution, whole channel tile.  A thread's fragments lie on 4 pixel rows; the residual pairs of ROWS
// of them are loaded into registers before the first store of those rows.  `out` and `res` are plain pointers that the
// compiler must assume to alias, so loads interleaved with stores would wait for one memory round trip per fragment (16
// per tile at NT = 32, 32 at NT = 64); this way a tile pays 4 / ROWS.  ROWS keeps the staged residual at 16 registers.  Nets never give an op's output the buffer of its
// residual (net.cu buffer planner), so the reordering cannot change a result.
template <int NT, typename RT, int ROWS = (NT / 8) * (int)sizeof(RT) <= 16 ? 4 : (NT / 8) * (int)sizeof(RT) <= 32 ? 2 : 1>
__device__ __forceinline__ void wg_epilogue_nhwc(const ConvParams& p, const float (&acc)[2][NT / 2], int n, int y0, int x0, int co0,
                                                 int w, int l, bool linear) {
  // row m = 64h + 16w + l/4 + 8e of the tile is pixel pix0 + (8h + e) * dpix of the frame: the thread's fragments sit at 4
  // pixel rows, and channel group j is a constant byte offset from them
  const int dpix = linear ? 8 : p.Wout;
  auto pix0 = [&](int frame) -> size_t {
    return linear ? ((size_t)frame * p.Hout + y0) * p.Wout + x0 + 16 * w + (l >> 2)
                  : ((size_t)frame * p.Hout + y0 + 2 * w) * p.Wout + x0 + (l >> 2);
  };
  const int c = co0 + 2 * (l & 3);
  const uint8_t* rbase = nullptr;
  int rstep = 0;
  if (p.res != nullptr) {
    rbase = reinterpret_cast<const uint8_t*>(p.res) + (pix0(p.res_broadcast ? 0 : n) * p.res_C + p.res_c_off + c) * (sizeof(RT) / 2);
    rstep = dpix * p.res_C * (int)(sizeof(RT) / 2);
  }
  const int ob = p.out_dtype == B200ROMP_BF16 ? 2 : 4;
  uint8_t* obase = reinterpret_cast<uint8_t*>(p.out) + (pix0(n) * p.out_C + p.out_c_off + c) * ob;
  const int ostep = dpix * p.out_C * ob;
#pragma unroll
  for (int q0 = 0; q0 < 4; q0 += ROWS) {   // fragment row q = 2h + e
    RT rv[ROWS][NT / 8];
    if (p.res != nullptr) {
#pragma unroll
      for (int qq = 0; qq < ROWS; ++qq) {
        const int q = q0 + qq;
        const RT* r = reinterpret_cast<const RT*>(rbase + (8 * (q >> 1) + (q & 1)) * rstep);
#pragma unroll
        for (int j = 0; j < NT / 8; ++j) rv[qq][j] = r[4 * j];   // channel 8j: RT holds 2 channels
      }
    }
#pragma unroll
    for (int qq = 0; qq < ROWS; ++qq) {
      const int q = q0 + qq, h = q >> 1, e = q & 1;
      uint8_t* o = obase + (8 * h + e) * ostep;
#pragma unroll
      for (int j = 0; j < NT / 8; ++j) {
        float a = acc[h][4 * j + 2 * e], b = acc[h][4 * j + 2 * e + 1];   // bias included
        if (p.res != nullptr) { const float2 r = res_pair(rv[qq][j]); a += r.x; b += r.y; }
        if (p.relu) { a = fmaxf(a, 0.f); b = fmaxf(b, 0.f); }
        if (ob == 2) reinterpret_cast<__nv_bfloat162*>(o)[4 * j] = __floats2bfloat162_rn(a, b);
        else reinterpret_cast<float2*>(o)[4 * j] = make_float2(a, b);
      }
    }
  }
}

// Epilogue of one 128-pixel x NT-channel tile held as two m64 accumulators (rows 0-63 / 64-127) by a warpgroup: row m of the
// tile is pixel (m / 8, m % 8) of the 16 x 8 tile at (y0, x0) of frame n (linear: pixel (y0, x0 + m), a 128-wide row).  wgmma fragment: thread (warp w, lane l) holds,
// for each 8-column group j, columns 8j + 2(l%4) + {0,1} of rows 16w + l/4 (regs 4j, 4j+1) and 16w + l/4 + 8 (4j+2, 4j+3).
// The accumulators are consumed: the bias is added in place.  PATH selects the code compiled in: kEpiNhwc when the caller
// guarantees an NHWC conv-resolution output (tc_nhwc_out), kEpiGeneric when it guarantees the opposite, kEpiAny decides per
// tile.  A kernel that carries both needs about 40 registers more than one with kEpiNhwc alone.
constexpr int kEpiNhwc = 0, kEpiGeneric = 1, kEpiAny = 2;
template <int NT, int PATH = kEpiAny>
__device__ __forceinline__ void wg_epilogue(const ConvParams& p, float (&acc)[2][NT / 2], const float* __restrict__ bias, int n,
                                            int y0, int x0, int co0, int wg_thread, bool linear = false) {
  const int w = wg_thread >> 5, l = wg_thread & 31;
  if (PATH == kEpiNhwc || (PATH == kEpiAny && tc_nhwc_out(p, co0 + NT))) {
#pragma unroll
    for (int j = 0; j < NT / 8; ++j) {
      const int c = co0 + 8 * j + 2 * (l & 3);
      const float b0 = __ldg(bias + c), b1 = __ldg(bias + c + 1);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        acc[h][4 * j] += b0; acc[h][4 * j + 1] += b1; acc[h][4 * j + 2] += b0; acc[h][4 * j + 3] += b1;
      }
    }
    if (p.res != nullptr && p.res_dtype == B200ROMP_F32) wg_epilogue_nhwc<NT, float2>(p, acc, n, y0, x0, co0, w, l, linear);
    else wg_epilogue_nhwc<NT, uint32_t>(p, acc, n, y0, x0, co0, w, l, linear);
    return;
  }
  if constexpr (PATH != kEpiNhwc) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
#pragma unroll
      for (int j = 0; j < NT / 8; ++j) {
        const int c = co0 + 8 * j + 2 * (l & 3);
        const float b0 = __ldg(bias + c), b1 = __ldg(bias + c + 1);
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int m = 64 * h + 16 * w + (l >> 2) + 8 * e;
          wg_store2(p, n, linear ? y0 : y0 + (m >> 3), linear ? x0 + m : x0 + (m & 7), c, acc[h][4 * j + 2 * e] + b0,
                    acc[h][4 * j + 2 * e + 1] + b1);
        }
      }
    }
  }
}

// Epilogue of the swapped 3x3 plan (conv_tc.cu SWAP): one 64-channel x 128-pixel accumulator, channel-major.  Thread (warp
// w, lane l) holds channels co0 + 16w + l/4 + 8e of pixels 8j + 2 (l % 4) + {0, 1} (registers 4j + 2e + {0, 1}); pixel
// 8j + i of the tile is (y0 + j, x0 + i) of frame n.  Lanes l and l ^ 4 hold channels c and c ^ 1 of the same pixels and
// swap one fp32 value per pair, so each lane then holds 2 adjacent channels of one pixel and a warp's store covers 16 B of
// each of 8 pixels, as in wg_epilogue_nhwc.  Bias, residual and ReLU are applied to the same fp32 values in the same order
// as wg_epilogue, so the bf16 output is bit-identical.  Output bf16 NHWC at conv resolution; residual bf16 (RT = uint32_t,
// 2 channels) or fp32 (RT = float2), optionally broadcast from frame 0.  The residuals of JB tile rows are loaded before
// those rows' stores (see wg_epilogue_nhwc on aliasing); JB keeps them at 32 registers.
template <typename RT, int JB = sizeof(RT) == 4 ? 16 : 8>
__device__ __forceinline__ void wg_epilogue_swap(const ConvParams& p, const float (&acc)[64], int n, int y0, int x0, int co0,
                                                 int wg_thread) {
  const int w = wg_thread >> 5, l = wg_thread & 31, odd = (l >> 2) & 1;
  const int c = co0 + 16 * w + (l >> 2);           // this lane's accumulator channel for e = 0 (c + 8 for e = 1)
  const float bias[2] = {__ldg(p.bias + c), __ldg(p.bias + c + 8)};
  const int ch = c & ~1;                            // the first of the 2 channels this lane stores
  const size_t pix = ((size_t)n * p.Hout + y0) * p.Wout + x0 + 2 * (l & 3) + odd;   // the pixel it stores, tile row 0
  __nv_bfloat16* out = reinterpret_cast<__nv_bfloat16*>(p.out) + pix * p.out_C + p.out_c_off + ch;
  const size_t ostep = (size_t)p.Wout * p.out_C;
  const uint8_t* rbase = nullptr;
  size_t rstep = 0;
  if (p.res != nullptr) {
    const size_t rpix = p.res_broadcast ? pix - (size_t)n * p.Hout * p.Wout : pix;
    rbase = reinterpret_cast<const uint8_t*>(p.res) + (rpix * p.res_C + p.res_c_off + ch) * (sizeof(RT) / 2);
    rstep = (size_t)p.Wout * p.res_C * (sizeof(RT) / 2);
  }
#pragma unroll
  for (int j0 = 0; j0 < 16; j0 += JB) {
    RT rv[JB][2];
    if (p.res != nullptr) {
#pragma unroll
      for (int jj = 0; jj < JB; ++jj)
#pragma unroll
        for (int e = 0; e < 2; ++e) rv[jj][e] = reinterpret_cast<const RT*>(rbase + (j0 + jj) * rstep)[4 * e];   // channel + 8e
    }
#pragma unroll
    for (int jj = 0; jj < JB; ++jj) {
      const int j = j0 + jj;
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const float v0 = acc[4 * j + 2 * e] + bias[e], v1 = acc[4 * j + 2 * e + 1] + bias[e];
        // even lanes keep pixel 0 and send pixel 1, odd lanes the other way round
        const float recv = __shfl_xor_sync(0xffffffffu, odd ? v0 : v1, 4);
        float a = odd ? recv : v0, b = odd ? v1 : recv;
        if (p.res != nullptr) { const float2 r = res_pair(rv[jj][e]); a += r.x; b += r.y; }
        if (p.relu) { a = fmaxf(a, 0.f); b = fmaxf(b, 0.f); }
        *reinterpret_cast<__nv_bfloat162*>(out + j * ostep + 8 * e) = __floats2bfloat162_rn(a, b);
      }
    }
  }
}

// launch with the programmatic-stream-serialization attribute (see pdl_trigger / pdl_wait); B200ROMP_NO_PDL=1 disables it
template <typename... KArgs, typename... Args>
static inline cudaError_t tc_launch(void (*kern)(KArgs...), dim3 grid, int threads, int smem_bytes, cudaStream_t stream, Args&&... args) {
  static const bool pdl_default = [] { const char* e = getenv("B200ROMP_NO_PDL"); return !(e && e[0] == '1'); }();
  const bool pdl = pdl_default && g_tc_pdl_override != 0;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = dim3(threads);
  cfg.dynamicSmemBytes = (size_t)smem_bytes;
  cfg.stream = stream;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at;
  cfg.numAttrs = pdl ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
}

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                    const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
PFN_encodeTiled tc_get_encode();
// A tiled TMA map over a `rank`-dimensional tensor at `base`: element dims, byte strides of dims 1 .. rank-1, box, element
// strides 1, 128 B L2 promotion, zeros outside the tensor.  On failure the error text starts with `tag`.
int tc_encode_tiled(CUtensorMap* map, CUtensorMapDataType dtype, int rank, const void* base, const cuuint64_t* dims,
                    const cuuint64_t* strides, const cuuint32_t* box, CUtensorMapSwizzle swizzle, const char* tag);
// the map over the NHWC input channel slice [in_c_off, in_c_off + cin) of `p` in bf16 (eb = 2) or fp32 (eb = 4): dims
// (cin, W, H, N) and a (box_c, box_w, box_h, 1) halo box whose out-of-bounds pixels read as zeros
int tc_encode_nhwc_input(CUtensorMap* map, const ConvParams& p, int eb, int box_c, int box_w, int box_h, CUtensorMapSwizzle swizzle,
                         const char* tag);
// bf16 / TF32 weight slab in shared-memory-image order [ntile][tap][chunk][NT rows x ROWB] with the TMA / wgmma XOR swizzle:
// tc_pack_image builds it on the host, tc_pack_weights uploads it as well
std::vector<uint8_t> tc_pack_image(const float* w_oihw, int cin, int cout, int taps, int nt, int rowb, int eb);
int tc_pack_weights(const float* w_oihw, int cin, int cout, int taps, int nt, void** d_out, std::vector<void*>* allocs, int rowb, int eb);
float tc_round_tf32_host(float w);   // fp32 -> TF32, ties away from zero (cvt.rna.tf32.f32)

}  // namespace b200romp
