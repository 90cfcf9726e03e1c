// Shared helpers for libb200romp (sm_90a).  Internal header - not part of the C ABI.
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <stdio.h>
#include <string>
#include <vector>

#include "../../include/b200romp.h"

namespace b200romp {

void set_error(const char* fmt, ...);
// copies `bytes` of host memory to a new device allocation, recorded in `allocs`; nullptr (error set) on failure
void* upload(const void* host, size_t bytes, std::vector<void*>* allocs);
// -1 = default; 0 = launch the next tensor-core convs without the programmatic-dependent-launch attribute (net.cu: ops that wait
// for another lane inside the captured graph).  Defined in conv_tc.cu.
extern thread_local int g_tc_pdl_override;

#define B2R_CUDA_OK(expr)                                                                         \
  do {                                                                                            \
    cudaError_t _e = (expr);                                                                      \
    if (_e != cudaSuccess) {                                                                      \
      ::b200romp::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
      return B200ROMP_ECUDA;                                                                      \
    }                                                                                             \
  } while (0)

#define B2R_REQUIRE(cond, ...)                 \
  do {                                         \
    if (!(cond)) {                             \
      ::b200romp::set_error(__VA_ARGS__);      \
      return B200ROMP_EINVAL;                  \
    }                                          \
  } while (0)

static inline size_t dtype_size(int dt) { return dt == B200ROMP_F32 ? 4 : (dt == B200ROMP_BF16 ? 2 : 1); }

// Device-side description of one fused conv op (see b200romp_conv_desc in the public header).
struct ConvParams {
  const void* in;
  void* out;
  const void* res;
  const float* w;     // SIMT packing: [tap][cin][coutPad] fp32
  const float* bias;  // [coutPad] fp32 (zeros when the layer has no bias)
  int B;
  int Hin, Win, in_C, in_c_off, cin;
  int Hout, Wout;            // conv output grid (before upsampling)
  int out_C, out_c_off, cout, coutPad;
  int up;                    // nearest upsample factor; full-res grid is Hout*up x Wout*up
  int res_C, res_c_off, res_broadcast;
  int relu, pow_channel, out_nchw;
  int in_dtype, out_dtype, res_dtype;
  int input_norm;
};

// ---- epilogue shared by the SIMT and tensor-core conv kernels ---------------------------------------
__device__ __forceinline__ float load_as_float(const void* p, size_t idx, int dt) {
  return dt == B200ROMP_F32 ? reinterpret_cast<const float*>(p)[idx]
                            : __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(p)[idx]);
}

__device__ __forceinline__ void store_from_float(void* p, size_t idx, int dt, float v) {
  if (dt == B200ROMP_F32) reinterpret_cast<float*>(p)[idx] = v;
  else reinterpret_cast<__nv_bfloat16*>(p)[idx] = __float2bfloat16_rn(v);
}

// Finish NV consecutive output channels [co, co+NV) of conv-output pixel (n, oy, ox): bias is already
// added by the caller.  Handles residual, ReLU, 1.1**x, upsample replication, NHWC/NCHW and dtypes.
template <int NV>
__device__ __forceinline__ void conv_epilogue_store(const ConvParams& p, int n, int oy, int ox, int co,
                                                    const float (&v)[NV]) {
  const int Hf = p.Hout * p.up, Wf = p.Wout * p.up;
  const bool vec_ok = (NV % 4 == 0) && !p.out_nchw && (co + NV <= p.cout) && ((p.out_C | p.out_c_off) % 4 == 0) &&
                      (p.res == nullptr || ((p.res_C | p.res_c_off) % 4 == 0)) && p.pow_channel < 0;
  for (int dy = 0; dy < p.up; ++dy) {
    for (int dx = 0; dx < p.up; ++dx) {
      const int fy = oy * p.up + dy, fx = ox * p.up + dx;
      const size_t pix = ((size_t)n * Hf + fy) * Wf + fx;
      const size_t rpix = ((size_t)(p.res_broadcast ? 0 : n) * Hf + fy) * Wf + fx;
      if (vec_ok) {
#pragma unroll
        for (int q = 0; q < NV; q += 4) {
          float o[4] = {v[q], v[q + 1], v[q + 2], v[q + 3]};
          if (p.res != nullptr) {
            const size_t ri = rpix * p.res_C + p.res_c_off + co + q;
            if (p.res_dtype == B200ROMP_F32) {
              const float4 r = *reinterpret_cast<const float4*>(reinterpret_cast<const float*>(p.res) + ri);
              o[0] += r.x; o[1] += r.y; o[2] += r.z; o[3] += r.w;
            } else {
              const uint2 r = *reinterpret_cast<const uint2*>(reinterpret_cast<const __nv_bfloat16*>(p.res) + ri);
              const __nv_bfloat162 r01 = *reinterpret_cast<const __nv_bfloat162*>(&r.x);
              const __nv_bfloat162 r23 = *reinterpret_cast<const __nv_bfloat162*>(&r.y);
              o[0] += __low2float(r01); o[1] += __high2float(r01);
              o[2] += __low2float(r23); o[3] += __high2float(r23);
            }
          }
          if (p.relu) {
#pragma unroll
            for (int j = 0; j < 4; ++j) o[j] = fmaxf(o[j], 0.f);
          }
          const size_t oi = pix * p.out_C + p.out_c_off + co + q;
          if (p.out_dtype == B200ROMP_F32) {
            *reinterpret_cast<float4*>(reinterpret_cast<float*>(p.out) + oi) = make_float4(o[0], o[1], o[2], o[3]);
          } else {
            __nv_bfloat162 a = __floats2bfloat162_rn(o[0], o[1]);
            __nv_bfloat162 b = __floats2bfloat162_rn(o[2], o[3]);
            uint2 pk;
            pk.x = *reinterpret_cast<uint32_t*>(&a);
            pk.y = *reinterpret_cast<uint32_t*>(&b);
            *reinterpret_cast<uint2*>(reinterpret_cast<__nv_bfloat16*>(p.out) + oi) = pk;
          }
        }
      } else {
#pragma unroll
        for (int q = 0; q < NV; ++q) {
          const int c = co + q;
          if (c >= p.cout) break;
          float o = v[q];
          if (p.res != nullptr) o += load_as_float(p.res, rpix * p.res_C + p.res_c_off + c, p.res_dtype);
          if (p.relu) o = fmaxf(o, 0.f);
          if (c == p.pow_channel) o = powf(1.1f, o);
          const size_t oi = p.out_nchw ? (((size_t)n * p.out_C + p.out_c_off + c) * Hf + fy) * Wf + fx
                                       : pix * p.out_C + p.out_c_off + c;
          store_from_float(p.out, oi, p.out_dtype, o);
        }
      }
    }
  }
}

// fuse-layer sum op (conv_simt.cu)
struct SumParams {
  const void* base;
  const void* term[4];
  void* out;
  int base_dt, term_dt[4], out_dt;
  int n_terms, up[4];
  int term_C[4], term_c_off[4];   // channels of the term tensors (>= C) and the first channel of the slice that is added
  int B, H, W, C, relu;
};
int launch_fuse_sum(const SumParams& p, cudaStream_t stream);
// the kernel launch_fuse_sum takes for p ("ring", "pipe" or "simple"): it depends on the pointers' alignment, so p must be bound
const char* fuse_sum_kernel_name(const SumParams& p);

// engines implemented in other translation units
int launch_conv_simt(const ConvParams& p, int ksize, int stride, cudaStream_t stream);
// ResNet-50 variant only (resnet_ops.cu): generic k x k conv (7x7 stem), ConvTranspose2d(4,2,1), MaxPool2d(3,2,1)
int launch_conv_generic(const ConvParams& p, int ksize, int stride, cudaStream_t stream);
int launch_deconv4x4s2(const ConvParams& p, cudaStream_t stream);
int launch_maxpool3x3s2(const void* in, void* out, int dtype, int B, int Hin, int Win, int C, cudaStream_t stream);
// conv-output geometry for a ksize code: 1 / 3 / 7 = square kernels (pad k/2), 13 = Conv1d 1x3, 42 = ConvTranspose2d(4,2,1)
static inline void conv_out_hw(int ksize, int stride, int H, int W, int* Ho, int* Wo) {
  if (ksize == 42) { *Ho = 2 * H; *Wo = 2 * W; return; }
  const int kh = ksize == 13 ? 1 : ksize, kw = ksize == 13 ? 3 : ksize;
  *Ho = (H + 2 * (kh / 2) - kh) / stride + 1;
  *Wo = (W + 2 * (kw / 2) - kw) / stride + 1;
}
static inline int conv_taps(int ksize) { return ksize == 13 ? 3 : (ksize == 42 ? 16 : ksize * ksize); }

}  // namespace b200romp
