// Generic fused direct convolution on CUDA cores (fp32 accumulate).
//
// Role: (1) the fp32 "parity" engine - bit-for-bit the reference's arithmetic type (model.py convs run
// fp32), used to prove graph/BN-fold/fuse semantics against the oracle; (2) the engine for the few
// layers whose shapes do not map onto tensor-core tiles (3-channel stem, 142/3/1-channel head outputs).
// The dominant layers run on the wgmma implicit-GEMM engine in conv_tc.cu.
//
// Replaces per layer: nn.Conv2d + nn.BatchNorm2d (folded) + ReLU + residual add + nn.Upsample(nearest)
// (simple_romp/romp/model.py:49-83,85-123,185-244,338-343,449-466) and the input normalisation of
// model.py:384.
//
// Tiling: one CTA = 8x8 output pixels x 64 output channels, 256 threads, each thread a 4(pixel) x
// 4(channel) register tile; input halo tile and weight slab staged in shared memory in chunks of 8
// input channels.  HBM/L2 traffic per CTA: input halo once per 64-channel slab, weights once per tile.
#include <algorithm>

#include "common.cuh"
#include "conv_tc.cuh"
#include "tc_device.cuh"   // mbarrier / bulk-copy helpers for the fuse-sum ring

namespace b200romp {

enum { IN_F32 = 0, IN_BF16 = 1, IN_U8 = 2 };

template <int KH, int KW, int STRIDE>
__global__ void __launch_bounds__(256) conv_simt_kernel(const ConvParams p) {
  constexpr int TS = 8;
  constexpr int ITH = (TS - 1) * STRIDE + KH, ITW = (TS - 1) * STRIDE + KW;
  constexpr int KC = 8;
  constexpr int PADH = KH / 2, PADW = KW / 2;
  __shared__ float s_in[ITH * ITW][KC + 1];
  __shared__ __align__(16) float s_w[KH * KW][KC][64];

  const int tid = threadIdx.x;
  const int tilesX = (p.Wout + TS - 1) / TS;
  const int oy0 = (blockIdx.x / tilesX) * TS, ox0 = (blockIdx.x % tilesX) * TS;
  const int co0 = blockIdx.y * 64;
  const int n = blockIdx.z;
  const int tc = tid & 15, tp = tid >> 4;
  const int prow = tp >> 1, pcol = (tp & 1) * 4;

  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  const int iy0 = oy0 * STRIDE - PADH, ix0 = ox0 * STRIDE - PADW;
  for (int c0 = 0; c0 < p.cin; c0 += KC) {
    for (int idx = tid; idx < ITH * ITW * KC; idx += 256) {
      const int ci = idx % KC, pix = idx / KC;
      const int gy = iy0 + pix / ITW, gx = ix0 + pix % ITW;
      float v = 0.f;
      if (gy >= 0 && gy < p.Hin && gx >= 0 && gx < p.Win && c0 + ci < p.cin) {
        const size_t gi = (((size_t)n * p.Hin + gy) * p.Win + gx) * p.in_C + p.in_c_off + c0 + ci;
        if (p.in_dtype == IN_F32) v = reinterpret_cast<const float*>(p.in)[gi];
        else if (p.in_dtype == IN_BF16) v = __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(p.in)[gi]);
        else v = (float)reinterpret_cast<const unsigned char*>(p.in)[gi];
        if (p.input_norm) v = (v / 255.f) * 2.f - 1.f;   // model.py:384, same op order
      }
      s_in[pix][ci] = v;
    }
    for (int idx = tid; idx < KH * KW * KC * 64; idx += 256) {
      const int co = idx & 63, ci = (idx >> 6) % KC, tap = idx / (64 * KC);
      float v = 0.f;
      if (c0 + ci < p.cin) v = p.w[((size_t)tap * p.cin + c0 + ci) * p.coutPad + co0 + co];
      s_w[tap][ci][co] = v;
    }
    __syncthreads();
#pragma unroll
    for (int ky = 0; ky < KH; ++ky) {
#pragma unroll
      for (int kx = 0; kx < KW; ++kx) {
#pragma unroll
        for (int ci = 0; ci < KC; ++ci) {
          const float4 w4 = *reinterpret_cast<const float4*>(&s_w[ky * KW + kx][ci][tc * 4]);
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const float a = s_in[(prow * STRIDE + ky) * ITW + (pcol + i) * STRIDE + kx][ci];
            acc[i][0] = fmaf(a, w4.x, acc[i][0]);
            acc[i][1] = fmaf(a, w4.y, acc[i][1]);
            acc[i][2] = fmaf(a, w4.z, acc[i][2]);
            acc[i][3] = fmaf(a, w4.w, acc[i][3]);
          }
        }
      }
    }
    __syncthreads();
  }

  const int co = co0 + tc * 4;
  if (co >= p.cout) return;
  float b[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) b[j] = p.bias[co + j];   // bias is padded to coutPad
  const int oy = oy0 + prow;
  if (oy >= p.Hout) return;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int ox = ox0 + pcol + i;
    if (ox >= p.Wout) continue;
    float v[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) v[j] = acc[i][j] + b[j];
    conv_epilogue_store<4>(p, n, oy, ox, co, v);
  }
}

// ------------------------------------------------------------------------------------------------
// Stem: 3x3 stride-2 conv on the raw 3-channel frames (model.py:338-340,384-387).  HBM-bound in principle
// (0.79 MB u8 in, 8.4 MB bf16 out per frame); K = 27 is too thin for a tensor-core tile, so: CTA = 8 x 32 output
// pixels, one thread per pixel, all 64 channels in registers 16 at a time; the normalised input tile is staged in
// shared memory with even/odd columns de-interleaved so that the stride-2 reads are bank-conflict free, and the
// 27 x 64 weights are read as broadcast float4.  Output: 128 contiguous bytes per thread, 16-byte stores.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) conv_stem_kernel(const ConvParams p) {
  constexpr int TW = 32, TH = 8, IH = 2 * TH + 1, HALF = TW + 1;
  __shared__ float s_in[IH][2][HALF][3];
  __shared__ __align__(16) float s_w[27][64];
  __shared__ float s_b[64];
  const int tid = threadIdx.x;
  const int ox0 = blockIdx.x * TW, oy0 = blockIdx.y * TH, n = blockIdx.z;
  const int iy0 = 2 * oy0 - 1, ix0 = 2 * ox0 - 1;
  for (int idx = tid; idx < IH * (2 * HALF - 1) * 3; idx += 256) {
    const int c = idx % 3, ix = (idx / 3) % (2 * HALF - 1), iy = idx / (3 * (2 * HALF - 1));
    const int gy = iy0 + iy, gx = ix0 + ix;
    float v = 0.f;
    if (gy >= 0 && gy < p.Hin && gx >= 0 && gx < p.Win) {
      const size_t gi = (((size_t)n * p.Hin + gy) * p.Win + gx) * p.in_C + p.in_c_off + c;
      if (p.in_dtype == IN_F32) v = reinterpret_cast<const float*>(p.in)[gi];
      else if (p.in_dtype == IN_BF16) v = __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(p.in)[gi]);
      else v = (float)reinterpret_cast<const unsigned char*>(p.in)[gi];
      if (p.input_norm) v = (v / 255.f) * 2.f - 1.f;
    }
    s_in[iy][ix & 1][ix >> 1][c] = v;
  }
  for (int idx = tid; idx < 27 * 64; idx += 256) {
    const int co = idx & 63, k = idx >> 6;                 // k = tap*3 + ci, SIMT packing [tap][cin][coutPad]
    s_w[k][co] = co < p.cout ? p.w[(size_t)k * p.coutPad + co] : 0.f;
  }
  if (tid < 64) s_b[tid] = p.bias[tid];
  __syncthreads();
  const int tx = tid & 31, ty = tid >> 5;
  const int oy = oy0 + ty, ox = ox0 + tx;
  float a[27];
#pragma unroll
  for (int ky = 0; ky < 3; ++ky)
#pragma unroll
    for (int kx = 0; kx < 3; ++kx)
#pragma unroll
      for (int c = 0; c < 3; ++c) a[(ky * 3 + kx) * 3 + c] = s_in[2 * ty + ky][kx & 1][tx + (kx >> 1)][c];
  if (oy >= p.Hout || ox >= p.Wout) return;
  const size_t pix = ((size_t)n * p.Hout + oy) * p.Wout + ox;
  for (int cg = 0; cg < p.cout; cg += 16) {
    float acc[16];
#pragma unroll
    for (int j = 0; j < 16; ++j) acc[j] = s_b[cg + j];
#pragma unroll
    for (int k = 0; k < 27; ++k) {
#pragma unroll
      for (int g = 0; g < 4; ++g) {
        const float4 w4 = *reinterpret_cast<const float4*>(&s_w[k][cg + g * 4]);
        acc[g * 4 + 0] = fmaf(a[k], w4.x, acc[g * 4 + 0]);
        acc[g * 4 + 1] = fmaf(a[k], w4.y, acc[g * 4 + 1]);
        acc[g * 4 + 2] = fmaf(a[k], w4.z, acc[g * 4 + 2]);
        acc[g * 4 + 3] = fmaf(a[k], w4.w, acc[g * 4 + 3]);
      }
    }
    if (p.relu) {
#pragma unroll
      for (int j = 0; j < 16; ++j) acc[j] = fmaxf(acc[j], 0.f);
    }
    const size_t oi = pix * p.out_C + p.out_c_off + cg;
    if (p.out_dtype == B200ROMP_BF16) {
      uint4 pk[2];
      __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(pk);
#pragma unroll
      for (int j = 0; j < 8; ++j) h[j] = __floats2bfloat162_rn(acc[2 * j], acc[2 * j + 1]);
      uint4* o = reinterpret_cast<uint4*>(reinterpret_cast<__nv_bfloat16*>(p.out) + oi);
      o[0] = pk[0];
      o[1] = pk[1];
    } else {
      float4* o = reinterpret_cast<float4*>(reinterpret_cast<float*>(p.out) + oi);
#pragma unroll
      for (int g = 0; g < 4; ++g) o[g] = make_float4(acc[g * 4], acc[g * 4 + 1], acc[g * 4 + 2], acc[g * 4 + 3]);
    }
  }
}

static bool stem_eligible(const ConvParams& p, int ksize, int stride) {
  return ksize == 3 && stride == 2 && p.cin == 3 && p.cout <= 64 && p.cout % 16 == 0 && !p.out_nchw && p.res == nullptr &&
         p.up == 1 && p.pow_channel < 0 && p.out_C % 8 == 0 && p.out_c_off % 8 == 0;
}

int launch_conv_simt(const ConvParams& p, int ksize, int stride, cudaStream_t stream) {
  if (stem_eligible(p, ksize, stride)) {
    dim3 g((p.Wout + 31) / 32, (p.Hout + 7) / 8, p.B);
    conv_stem_kernel<<<g, 256, 0, stream>>>(p);
    B2R_CUDA_OK(cudaGetLastError());
    return B200ROMP_OK;
  }
  if (ksize == 13 && stride == 1 && p.up == 1) {
    // Conv1d(k=3) along W (bev/model.py:19-22): rows are independent, so the batch folds into the row index - unless the
    // residual is broadcast: its one frame is indexed by the row within a frame
    ConvParams q = p;
    if (!p.res_broadcast) { q.B = 1; q.Hin = p.B * p.Hin; q.Hout = p.B * p.Hout; }
    dim3 g(((q.Hout + 7) / 8) * ((q.Wout + 7) / 8), (q.cout + 63) / 64, q.B);
    conv_simt_kernel<1, 3, 1><<<g, 256, 0, stream>>>(q);
    B2R_CUDA_OK(cudaGetLastError());
    return B200ROMP_OK;
  }
  dim3 grid(((p.Hout + 7) / 8) * ((p.Wout + 7) / 8), (p.cout + 63) / 64, p.B);
  dim3 block(256);
  if (ksize == 3 && stride == 1) conv_simt_kernel<3, 3, 1><<<grid, block, 0, stream>>>(p);
  else if (ksize == 3 && stride == 2) conv_simt_kernel<3, 3, 2><<<grid, block, 0, stream>>>(p);
  else if (ksize == 1 && stride == 1) conv_simt_kernel<1, 1, 1><<<grid, block, 0, stream>>>(p);
  else if (ksize == 1 && stride == 2) conv_simt_kernel<1, 1, 2><<<grid, block, 0, stream>>>(p);
  else {
    set_error("conv_simt: unsupported ksize=%d stride=%d", ksize, stride);
    return B200ROMP_EINVAL;
  }
  B2R_CUDA_OK(cudaGetLastError());
  return B200ROMP_OK;
}

// ---- fuse-layer sum (b200romp_net_add_sum): HBM-bound elementwise op, thread = 8 channels of one output pixel -------
__device__ __forceinline__ void load8(const void* p, int dt, size_t idx, float (&v)[8]) {
  if (dt == B200ROMP_F32) {
    const float4 a = reinterpret_cast<const float4*>(reinterpret_cast<const float*>(p) + idx)[0];
    const float4 b = reinterpret_cast<const float4*>(reinterpret_cast<const float*>(p) + idx)[1];
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
  } else {
    const uint4 t = *reinterpret_cast<const uint4*>(reinterpret_cast<const __nv_bfloat16*>(p) + idx);
    const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&t);
#pragma unroll
    for (int k = 0; k < 4; ++k) { v[2 * k] = __low2float(h[k]); v[2 * k + 1] = __high2float(h[k]); }
  }
}

__device__ __forceinline__ void sum_finish_store(const SumParams& p, float (&s)[8], size_t oi) {
  if (p.relu) {
#pragma unroll
    for (int j = 0; j < 8; ++j) s[j] = fmaxf(s[j], 0.f);
  }
  if (p.out_dt == B200ROMP_F32) {
    float4* o = reinterpret_cast<float4*>(reinterpret_cast<float*>(p.out) + oi);
    o[0] = make_float4(s[0], s[1], s[2], s[3]);
    o[1] = make_float4(s[4], s[5], s[6], s[7]);
  } else {
    uint4 pk;
    __nv_bfloat162 h0 = __floats2bfloat162_rn(s[0], s[1]), h1 = __floats2bfloat162_rn(s[2], s[3]);
    __nv_bfloat162 h2 = __floats2bfloat162_rn(s[4], s[5]), h3 = __floats2bfloat162_rn(s[6], s[7]);
    pk.x = *reinterpret_cast<uint32_t*>(&h0); pk.y = *reinterpret_cast<uint32_t*>(&h1);
    pk.z = *reinterpret_cast<uint32_t*>(&h2); pk.w = *reinterpret_cast<uint32_t*>(&h3);
    *reinterpret_cast<uint4*>(reinterpret_cast<__nv_bfloat16*>(p.out) + oi) = pk;
  }
}

// Fallback: grid x = 16 B chunks of one output row (W * C/8), y = rows (B * H); one chunk per thread.
__global__ void __launch_bounds__(256) fuse_sum_kernel(const SumParams p, int c8n, int4 up_shift) {
  const int ush[4] = {up_shift.x, up_shift.y, up_shift.z, up_shift.w};
  for (int row = blockIdx.y; row < p.B * p.H; row += gridDim.y) {   // row = n * H + y
    const int n = row / p.H, y = row - n * p.H;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < p.W * c8n; i += gridDim.x * blockDim.x) {
      const int x = i / c8n, c8 = i - x * c8n;
      const size_t pix = (size_t)row * p.W + x;
      float s[8], t[8];
      load8(p.base, p.base_dt, pix * p.C + c8 * 8, s);
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        if (k < p.n_terms) {
          const int sh = ush[k];
          const size_t tp = ((size_t)n * (p.H >> sh) + (y >> sh)) * (p.W >> sh) + (x >> sh);
          load8(p.term[k], p.term_dt[k], tp * p.term_C[k] + p.term_c_off[k] + c8 * 8, t);
#pragma unroll
          for (int j = 0; j < 8; ++j) s[j] += t[j];
        }
      }
      sum_finish_store(p, s, pix * p.C + c8 * 8);
    }
  }
}

// Main version: persistent blocks stream the base tensor row by row through a kSumStages-deep shared-memory ring filled by
// 1-D bulk async copies (cp.async.bulk + mbarrier).  One 16 B load per thread keeps only ~32 KB per SM in flight; the ring keeps blocks/SM x stages x row bytes (~100 KB) in flight without spending registers.  The
// low-resolution terms are read with plain loads (re-used across up^2 outputs, L1/L2 hits).  DT = the one dtype of all
// tensors (the nets are all-bf16 or all-fp32), row pointers are hoisted and the inner loop is 32-bit arithmetic only:
// the first version spent ~245 instructions per 16 B chunk (ncu: issue slots 52 % busy, DRAM 35 %).
constexpr int kSumStages = 4;
template <int DT>
__device__ __forceinline__ void sum_load8(const void* p, uint32_t chunk, float (&v)[8]) {   // chunk = 8-element index
  if (DT == B200ROMP_F32) {
    const float4 a = reinterpret_cast<const float4*>(p)[2 * chunk], b = reinterpret_cast<const float4*>(p)[2 * chunk + 1];
    v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
  } else {
    const uint4 t = reinterpret_cast<const uint4*>(p)[chunk];
    const uint32_t w[4] = {t.x, t.y, t.z, t.w};
#pragma unroll
    for (int k = 0; k < 4; ++k) { v[2 * k] = __uint_as_float(w[k] << 16); v[2 * k + 1] = __uint_as_float(w[k] & 0xffff0000u); }
  }
}
// raw 8-element chunk: loads are issued first (registers: 4 for bf16, 8 for fp32), converted / accumulated later
template <int DT> struct SumRaw { uint4 a, b; };
template <int DT>
__device__ __forceinline__ void sum_load_raw(const void* p, uint32_t chunk, SumRaw<DT>& r) {
  if (DT == B200ROMP_F32) { r.a = reinterpret_cast<const uint4*>(p)[2 * chunk]; r.b = reinterpret_cast<const uint4*>(p)[2 * chunk + 1]; }
  else r.a = reinterpret_cast<const uint4*>(p)[chunk];
}
template <int DT>
__device__ __forceinline__ void sum_raw_to_float(const SumRaw<DT>& r, float (&v)[8]) {
  if (DT == B200ROMP_F32) {
    v[0] = __uint_as_float(r.a.x); v[1] = __uint_as_float(r.a.y); v[2] = __uint_as_float(r.a.z); v[3] = __uint_as_float(r.a.w);
    v[4] = __uint_as_float(r.b.x); v[5] = __uint_as_float(r.b.y); v[6] = __uint_as_float(r.b.z); v[7] = __uint_as_float(r.b.w);
  } else {
    const uint32_t w[4] = {r.a.x, r.a.y, r.a.z, r.a.w};
#pragma unroll
    for (int k = 0; k < 4; ++k) { v[2 * k] = __uint_as_float(w[k] << 16); v[2 * k + 1] = __uint_as_float(w[k] & 0xffff0000u); }
  }
}
template <int DT>
__global__ void __launch_bounds__(256, DT == B200ROMP_F32 ? 3 : 4) fuse_sum_pipe_kernel(const SumParams p, int c8n, int c8_shift, int4 up_shift, int row_bytes) {
  extern __shared__ uint8_t sum_smem_raw[];
  uint8_t* sm = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(sum_smem_raw) + 127) & ~(uintptr_t)127);
  uint64_t* full = reinterpret_cast<uint64_t*>(sm + (size_t)kSumStages * row_bytes);
  uint64_t* empty = full + kSumStages;
  const int ush[4] = {up_shift.x, up_shift.y, up_shift.z, up_shift.w};
  const int tc8n[4] = {p.term_C[0] >> 3, p.term_C[1] >> 3, p.term_C[2] >> 3, p.term_C[3] >> 3};   // 16 B chunks per term pixel
  const int rows = p.B * p.H, per_row = p.W * c8n;
  const int lane = threadIdx.x & 31;
  const uint8_t* base = reinterpret_cast<const uint8_t*>(p.base);
  constexpr int ES = DT == B200ROMP_F32 ? 4 : 2;
  if (threadIdx.x == 0) {
    for (int i = 0; i < kSumStages; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], blockDim.x / 32);
    }
    fence_barrier_init();
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int d = 0; d < kSumStages; ++d) {
      const int r = blockIdx.x + d * gridDim.x;
      if (r < rows) {
        mbar_arrive_expect_tx(&full[d], row_bytes);
        bulk_copy_g2s(sm + (size_t)d * row_bytes, base + (size_t)r * row_bytes, row_bytes, &full[d]);
      }
    }
  }
  int iter = 0;
  for (int row = blockIdx.x; row < rows; row += gridDim.x, ++iter) {
    const int st = iter % kSumStages;
    const uint32_t ph = (uint32_t)(iter / kSumStages) & 1u;
    const int n = row / p.H, y = row - n * p.H;
    const uint8_t* srow = sm + (size_t)st * row_bytes;
    const uint8_t* trow[4];                                  // term rows feeding this output row (start of the channel slice)
#pragma unroll
    for (int k = 0; k < 4; ++k)
      trow[k] = k < p.n_terms ? reinterpret_cast<const uint8_t*>(p.term[k]) +
                                    (((size_t)n * (p.H >> ush[k]) + (y >> ush[k])) * (size_t)(p.W >> ush[k]) * p.term_C[k] + p.term_c_off[k]) * ES
                              : nullptr;
    uint8_t* orow = reinterpret_cast<uint8_t*>(p.out) + (size_t)row * row_bytes;
    mbar_wait(&full[st], ph);
    // two chunks per thread and trip: all loads of both chunks are issued before the first store (the output may alias
    // nothing, but the compiler cannot know) - twice the bytes in flight per warp (ncu: long-scoreboard bound)
    constexpr int U = DT == B200ROMP_F32 ? 1 : 2;           // fp32 chunks are twice the registers: one per trip
    for (int i0 = threadIdx.x; i0 < per_row; i0 += U * blockDim.x) {
      const int i1 = i0 + blockDim.x;
      const bool two = U == 2 && i1 < per_row;
      SumRaw<DT> rb[U], rt[U][4];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int i = u ? i1 : i0;
        if (u && !two) break;
        const int x = c8_shift >= 0 ? (i >> c8_shift) : i / c8n, c8 = i - x * c8n;
        sum_load_raw<DT>(srow, i, rb[u]);                   // generic load from shared memory
#pragma unroll
        for (int k = 0; k < 4; ++k)
          if (k < p.n_terms) sum_load_raw<DT>(trow[k], (uint32_t)((x >> ush[k]) * tc8n[k] + c8), rt[u][k]);
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int i = u ? i1 : i0;
        if (u && !two) break;
        float s[1][8], t[8];
        sum_raw_to_float<DT>(rb[u], s[0]);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          if (k < p.n_terms) {
            sum_raw_to_float<DT>(rt[u][k], t);
#pragma unroll
            for (int j = 0; j < 8; ++j) s[0][j] += t[j];     // order: base, term 0, 1, ...
          }
        }
        if (p.relu) {
#pragma unroll
          for (int j = 0; j < 8; ++j) s[0][j] = fmaxf(s[0][j], 0.f);
        }
        if (DT == B200ROMP_F32) {
          reinterpret_cast<float4*>(orow)[2 * i] = make_float4(s[0][0], s[0][1], s[0][2], s[0][3]);
          reinterpret_cast<float4*>(orow)[2 * i + 1] = make_float4(s[0][4], s[0][5], s[0][6], s[0][7]);
        } else {
          uint4 pk;
          __nv_bfloat162 h0 = __floats2bfloat162_rn(s[0][0], s[0][1]), h1 = __floats2bfloat162_rn(s[0][2], s[0][3]);
          __nv_bfloat162 h2 = __floats2bfloat162_rn(s[0][4], s[0][5]), h3 = __floats2bfloat162_rn(s[0][6], s[0][7]);
          pk.x = *reinterpret_cast<uint32_t*>(&h0); pk.y = *reinterpret_cast<uint32_t*>(&h1);
          pk.z = *reinterpret_cast<uint32_t*>(&h2); pk.w = *reinterpret_cast<uint32_t*>(&h3);
          reinterpret_cast<uint4*>(orow)[i] = pk;
        }
      }
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty[st]);
    if (threadIdx.x == 0) {
      const int next = row + kSumStages * gridDim.x;
      if (next < rows) {
        mbar_wait(&empty[st], ph);                          // every warp is done with this stage
        mbar_arrive_expect_tx(&full[st], row_bytes);
        bulk_copy_g2s(sm + (size_t)st * row_bytes, base + (size_t)next * row_bytes, row_bytes, &full[st]);
      }
    }
  }
}

// Ring version with the TERMS in the ring as well (B200ROMP_SUM_RING=1, for terms that are whole tensors): per output row the
// producer thread bulk-copies the base row and the term row of every term (rows of W/up pixels) into one stage; the compute
// loop then has no global load at all - in fuse_sum_pipe_kernel every row pays one exposed L2 round trip for its term loads
// (ncu: long-scoreboard 9 per issue, 2.9 TB/s).
struct SumRingCfg {
  int term_bytes[4];     // bytes of one term row
  int term_off[4];       // byte offset of term k inside a stage
  int stage_bytes, stages;
};
template <int DT>
__global__ void __launch_bounds__(256) fuse_sum_ring_kernel(const SumParams p, const SumRingCfg cfg, int c8n, int c8_shift, int4 up_shift,
                                                            int row_bytes) {
  extern __shared__ uint8_t sum_smem_raw[];
  uint8_t* sm = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(sum_smem_raw) + 127) & ~(uintptr_t)127);
  uint64_t* full = reinterpret_cast<uint64_t*>(sm + (size_t)cfg.stages * cfg.stage_bytes);
  uint64_t* empty = full + cfg.stages;
  const int ush[4] = {up_shift.x, up_shift.y, up_shift.z, up_shift.w};
  const int rows = p.B * p.H, per_row = p.W * c8n;
  const int lane = threadIdx.x & 31;
  constexpr int ES = DT == B200ROMP_F32 ? 4 : 2;
  if (threadIdx.x == 0) {
    for (int i = 0; i < cfg.stages; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], blockDim.x / 32);
    }
    fence_barrier_init();
  }
  __syncthreads();
  auto fill = [&](int r, int st) {     // thread 0: base row + one row of every term -> stage st
    const int n = r / p.H, y = r - n * p.H;
    int total = row_bytes;
    for (int k = 0; k < p.n_terms; ++k) total += cfg.term_bytes[k];
    uint8_t* dst = sm + (size_t)st * cfg.stage_bytes;
    mbar_arrive_expect_tx(&full[st], total);
    bulk_copy_g2s(dst, reinterpret_cast<const uint8_t*>(p.base) + (size_t)r * row_bytes, row_bytes, &full[st]);
    for (int k = 0; k < p.n_terms; ++k) {
      const size_t trow = (size_t)n * (p.H >> ush[k]) + (y >> ush[k]);
      bulk_copy_g2s(dst + cfg.term_off[k], reinterpret_cast<const uint8_t*>(p.term[k]) + trow * cfg.term_bytes[k], cfg.term_bytes[k], &full[st]);
    }
  };
  if (threadIdx.x == 0)
    for (int d = 0; d < cfg.stages; ++d) {
      const int r = blockIdx.x + d * gridDim.x;
      if (r < rows) fill(r, d);
    }
  int iter = 0;
  for (int row = blockIdx.x; row < rows; row += gridDim.x, ++iter) {
    const int st = iter % cfg.stages;
    const uint32_t ph = (uint32_t)(iter / cfg.stages) & 1u;
    const uint8_t* srow = sm + (size_t)st * cfg.stage_bytes;
    uint8_t* orow = reinterpret_cast<uint8_t*>(p.out) + (size_t)row * row_bytes;
    mbar_wait(&full[st], ph);
    for (int i = threadIdx.x; i < per_row; i += blockDim.x) {
      const int x = c8_shift >= 0 ? (i >> c8_shift) : i / c8n, c8 = i - x * c8n;
      float s[8], t[8];
      sum_load8<DT>(srow, i, s);
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        if (k < p.n_terms) {
          sum_load8<DT>(srow + cfg.term_off[k], (uint32_t)((x >> ush[k]) * c8n + c8), t);
#pragma unroll
          for (int j = 0; j < 8; ++j) s[j] += t[j];         // order: base, term 0, 1, ...
        }
      }
      if (p.relu) {
#pragma unroll
        for (int j = 0; j < 8; ++j) s[j] = fmaxf(s[j], 0.f);
      }
      if (DT == B200ROMP_F32) {
        reinterpret_cast<float4*>(orow)[2 * i] = make_float4(s[0], s[1], s[2], s[3]);
        reinterpret_cast<float4*>(orow)[2 * i + 1] = make_float4(s[4], s[5], s[6], s[7]);
      } else {
        uint4 pk;
        __nv_bfloat162 h0 = __floats2bfloat162_rn(s[0], s[1]), h1 = __floats2bfloat162_rn(s[2], s[3]);
        __nv_bfloat162 h2 = __floats2bfloat162_rn(s[4], s[5]), h3 = __floats2bfloat162_rn(s[6], s[7]);
        pk.x = *reinterpret_cast<uint32_t*>(&h0); pk.y = *reinterpret_cast<uint32_t*>(&h1);
        pk.z = *reinterpret_cast<uint32_t*>(&h2); pk.w = *reinterpret_cast<uint32_t*>(&h3);
        reinterpret_cast<uint4*>(orow)[i] = pk;
      }
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty[st]);
    if (threadIdx.x == 0) {
      const int next = row + cfg.stages * gridDim.x;
      if (next < rows) {
        mbar_wait(&empty[st], ph);                          // every warp is done with this stage
        fill(next, st);
      }
    }
  }
  (void)ES;
}

// Which fuse-sum kernel runs p: the pipe kernel when every tensor has the base's dtype and a base row fits the ring, the ring
// kernel instead when B200ROMP_SUM_RING=1 and every term is a whole tensor (no channel slice) with 16-byte rows (*ring then
// holds its stage layout), else the one-chunk-per-thread kernel (always with B200ROMP_SUM_SIMPLE=1).
enum class SumKernel { Simple, Pipe, Ring };
static SumKernel choose_fuse_sum(const SumParams& p, SumRingCfg* ring, int* ring_blocks_per_sm) {
  const int per_row = p.W * (p.C / 8);
  const int row_bytes = p.W * p.C * (int)dtype_size(p.base_dt);
  static const bool no_pipe = [] { const char* e = getenv("B200ROMP_SUM_SIMPLE"); return e && e[0] == '1'; }();
  bool same_dt = p.out_dt == p.base_dt;
  for (int k = 0; k < p.n_terms; ++k) same_dt = same_dt && p.term_dt[k] == p.base_dt;
  const bool pipe_ok = !no_pipe && same_dt && row_bytes % 16 == 0 && row_bytes <= 16384 && (reinterpret_cast<uintptr_t>(p.base) & 15) == 0 && per_row >= 128;
  if (!pipe_ok) return SumKernel::Simple;
  static const bool want_ring = [] { const char* e = getenv("B200ROMP_SUM_RING"); return e && e[0] == '1'; }();
  if (!want_ring) return SumKernel::Pipe;
  // every term a whole tensor (no channel slice) whose rows are 16-byte multiples: all operands travel through the ring
  SumRingCfg cfg;
  memset(&cfg, 0, sizeof(cfg));
  bool ok = true;
  int off = row_bytes;
  const int es = (int)dtype_size(p.base_dt);
  for (int k = 0; k < p.n_terms; ++k) {
    ok = ok && p.term_C[k] == p.C && p.term_c_off[k] == 0 && (reinterpret_cast<uintptr_t>(p.term[k]) & 15) == 0;
    cfg.term_bytes[k] = (p.W / p.up[k]) * p.C * es;
    ok = ok && cfg.term_bytes[k] % 16 == 0;
    cfg.term_off[k] = off;
    off += cfg.term_bytes[k];
  }
  cfg.stage_bytes = (off + 127) / 128 * 128;
  const int blocks_per_sm = cfg.stage_bytes <= 21 * 1024 ? 3 : 2;
  cfg.stages = std::min(4, (200 * 1024 / blocks_per_sm - 256) / cfg.stage_bytes);
  if (!ok || cfg.stages < 2) return SumKernel::Pipe;
  if (ring) *ring = cfg;
  if (ring_blocks_per_sm) *ring_blocks_per_sm = blocks_per_sm;
  return SumKernel::Ring;
}

const char* fuse_sum_kernel_name(const SumParams& p) {
  switch (choose_fuse_sum(p, nullptr, nullptr)) {
    case SumKernel::Ring: return "ring";
    case SumKernel::Pipe: return "pipe";
    default: return "simple";
  }
}

int launch_fuse_sum(const SumParams& p, cudaStream_t stream) {
  const int c8n = p.C / 8;
  auto lg = [](int u) { return u == 8 ? 3 : u == 4 ? 2 : u == 2 ? 1 : 0; };
  const int4 sh = make_int4(lg(p.up[0]), lg(p.up[1]), lg(p.up[2]), lg(p.up[3]));
  const int per_row = p.W * c8n;
  const int row_bytes = p.W * p.C * (int)dtype_size(p.base_dt);
  int c8_shift = -1;
  for (int b2 = 0; b2 < 8; ++b2) if ((1 << b2) == c8n) c8_shift = b2;
  SumRingCfg cfg;
  int ring_blocks_per_sm = 0;
  const SumKernel kernel = choose_fuse_sum(p, &cfg, &ring_blocks_per_sm);
  if (kernel == SumKernel::Ring) {
    const int smem = cfg.stages * cfg.stage_bytes + 2 * cfg.stages * 8 + 128;
    static bool ring_attr = false;
    if (!ring_attr) {
      B2R_CUDA_OK(cudaFuncSetAttribute(fuse_sum_ring_kernel<B200ROMP_F32>, cudaFuncAttributeMaxDynamicSharedMemorySize, 110 * 1024));
      B2R_CUDA_OK(cudaFuncSetAttribute(fuse_sum_ring_kernel<B200ROMP_BF16>, cudaFuncAttributeMaxDynamicSharedMemorySize, 110 * 1024));
      ring_attr = true;
    }
    const int grid = std::min(p.B * p.H, 132 * ring_blocks_per_sm);
    if (p.base_dt == B200ROMP_F32) fuse_sum_ring_kernel<B200ROMP_F32><<<grid, 256, smem, stream>>>(p, cfg, c8n, c8_shift, sh, row_bytes);
    else fuse_sum_ring_kernel<B200ROMP_BF16><<<grid, 256, smem, stream>>>(p, cfg, c8n, c8_shift, sh, row_bytes);
    B2R_CUDA_OK(cudaGetLastError());
    return B200ROMP_OK;
  }
  if (kernel == SumKernel::Pipe) {
    const int smem = kSumStages * row_bytes + 2 * kSumStages * 8 + 128;
    static bool attr_done = false;
    if (!attr_done) {
      B2R_CUDA_OK(cudaFuncSetAttribute(fuse_sum_pipe_kernel<B200ROMP_F32>, cudaFuncAttributeMaxDynamicSharedMemorySize, 4 * 16384 + 256));
      B2R_CUDA_OK(cudaFuncSetAttribute(fuse_sum_pipe_kernel<B200ROMP_BF16>, cudaFuncAttributeMaxDynamicSharedMemorySize, 4 * 16384 + 256));
      attr_done = true;
    }
    const int blocks_per_sm = row_bytes <= 8192 ? 4 : 3;
    const int grid = std::min(p.B * p.H, 132 * blocks_per_sm);
    if (p.base_dt == B200ROMP_F32) fuse_sum_pipe_kernel<B200ROMP_F32><<<grid, 256, smem, stream>>>(p, c8n, c8_shift, sh, row_bytes);
    else fuse_sum_pipe_kernel<B200ROMP_BF16><<<grid, 256, smem, stream>>>(p, c8n, c8_shift, sh, row_bytes);
    B2R_CUDA_OK(cudaGetLastError());
    return B200ROMP_OK;
  }
  const int threads = per_row >= 256 ? 256 : (per_row + 31) / 32 * 32;
  dim3 grid((per_row + threads - 1) / threads, std::min(p.B * p.H, 65535));
  fuse_sum_kernel<<<grid, threads, 0, stream>>>(p, c8n, sh);
  B2R_CUDA_OK(cudaGetLastError());
  return B200ROMP_OK;
}

}  // namespace b200romp
