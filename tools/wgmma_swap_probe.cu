// Does wgmma sum the same products in the same order when the operands swap roles?
//
// The fused BasicBlock (romp_b200/csrc/conv_block_tc.cu) must stay bit-identical to the unfused per-conv path, which runs
// every 3x3 conv as D[pixel][co] = X * W^T with the pixels as the A operand.  Issuing the weights as A and the pixels as B
// gives D^T; this probe checks, on seeded bf16 data, that D^T comes out bit for bit:
//   ref:  two m64n64k16 per k-step, A = X (64 pixels each), B = W
//   n128: one m64n128k16 per k-step, A = W, B = X (all 128 pixels)
//   n64:  two m64n64k16 per k-step, A = W, B = X (64 pixels each)
// each accumulated over 36 and 72 k-steps (9 / 18 taps x 4 k-steps of a 64-channel row, taps as shifted start addresses
// of a 20-pixel-wide halo as in the kernels, 128 B swizzle, scale_d = 0 on the first k-step and 1 after).
//
//   nvcc -std=c++17 -O3 -gencode arch=compute_90a,code=sm_90a -I romp_b200/csrc -o tools/wgmma_swap_probe tools/wgmma_swap_probe.cu
//   tools/wgmma_swap_probe            # exit code 0 iff every comparison is bit-identical
#include <cuda_bf16.h>

#include <cmath>
#include <cstdio>
#include <cstring>
#include <vector>

#include "tc_device.cuh"

using namespace b200romp;

namespace {

constexpr int kTrials = 8;
constexpr int kMaxTaps = 18;
constexpr int kHaloW = 20;
constexpr int kRowB = 128;                                  // 64 bf16 channels
constexpr int kTapShiftMax = (kMaxTaps / 3 - 1) * kHaloW + 2;
constexpr int kXRows = 128 + kTapShiftMax;
constexpr int kWBytes = kMaxTaps * 64 * kRowB;
constexpr int kXBytes = (kXRows * kRowB + 1023) / 1024 * 1024;
constexpr int kSmem = kWBytes + kXBytes + 1024;

__host__ __device__ constexpr int tap_shift(int tap) { return (tap / 3) * kHaloW + tap % 3; }

// one 64 x 128 B operand view with 8-row groups 1024 B apart, 128 B swizzle
__device__ __forceinline__ uint64_t desc(uint32_t addr) { return make_smem_desc(addr, 8 * kRowB, kSw128); }

// fragment register r of an m64 x N accumulator -> (row, column)
__device__ __forceinline__ void frag_rc(int t, int r, int& row, int& col) {
  const int w = t >> 5, l = t & 31, j = r >> 2, e = (r >> 1) & 1, b = r & 1;
  row = 16 * w + (l >> 2) + 8 * e;
  col = 8 * j + 2 * (l & 3) + b;
}

// one warpgroup per trial.  out: [trial][3][64 co][128 pixels] fp32 (ref is stored transposed, so all three compare alike)
__global__ void __launch_bounds__(128, 1) probe_kernel(const __nv_bfloat16* __restrict__ w, const __nv_bfloat16* __restrict__ x, int taps,
                                                      float* __restrict__ out) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* sW = smem;
  uint8_t* sX = smem + kWBytes;
  const int t = threadIdx.x, trial = blockIdx.x;
  const uint4* wg = reinterpret_cast<const uint4*>(w + (size_t)trial * kMaxTaps * 64 * 64);
  const uint4* xg = reinterpret_cast<const uint4*>(x + (size_t)trial * kXRows * 64);
  for (int i = t; i < kMaxTaps * 64 * 8; i += 128) {         // 16 B chunk c of row r goes to chunk c ^ (r & 7)
    const int r = i >> 3, c = i & 7;
    *reinterpret_cast<uint4*>(sW + r * kRowB + ((c ^ (r & 7)) << 4)) = wg[i];
  }
  for (int i = t; i < kXRows * 8; i += 128) {
    const int r = i >> 3, c = i & 7;
    *reinterpret_cast<uint4*>(sX + r * kRowB + ((c ^ (r & 7)) << 4)) = xg[i];
  }
  fence_proxy_async();
  __syncthreads();
  const uint32_t w0 = smem_u32(sW), x0 = smem_u32(sX);
  float* o = out + (size_t)trial * 3 * 64 * 128;
  const int steps = 4 * taps;

  {  // ref: A = X, B = W -> D[pixel][co]
    float d[2][32];
    uint32_t scale_d = 0;
    wgmma_fence();
    for (int s = 0; s < steps; ++s) {
      const int tap = s >> 2, k = s & 3;
      for (int h = 0; h < 2; ++h)
        wgmma_n64(d[h], desc(x0 + (tap_shift(tap) + 64 * h) * kRowB + 32 * k), desc(w0 + tap * 64 * kRowB + 32 * k), scale_d, false);
      scale_d = 1;
    }
    wgmma_commit();
    wgmma_wait<0>();
    for (int h = 0; h < 2; ++h)
      for (int r = 0; r < 32; ++r) {
        int row, col;
        frag_rc(t, r, row, col);
        o[col * 128 + 64 * h + row] = d[h][r];
      }
  }
  {  // n128: A = W, B = X -> D[co][pixel]
    float d[64];
    uint32_t scale_d = 0;
    wgmma_fence();
    for (int s = 0; s < steps; ++s) {
      const int tap = s >> 2, k = s & 3;
      wgmma_n128_bf16(d, desc(w0 + tap * 64 * kRowB + 32 * k), desc(x0 + tap_shift(tap) * kRowB + 32 * k), scale_d);
      scale_d = 1;
    }
    wgmma_commit();
    wgmma_wait<0>();
    for (int r = 0; r < 64; ++r) {
      int row, col;
      frag_rc(t, r, row, col);
      o[64 * 128 + row * 128 + col] = d[r];
    }
  }
  {  // n64: A = W, B = X, 64 pixels at a time
    float d[2][32];
    uint32_t scale_d = 0;
    wgmma_fence();
    for (int s = 0; s < steps; ++s) {
      const int tap = s >> 2, k = s & 3;
      for (int h = 0; h < 2; ++h)
        wgmma_n64(d[h], desc(w0 + tap * 64 * kRowB + 32 * k), desc(x0 + (tap_shift(tap) + 64 * h) * kRowB + 32 * k), scale_d, false);
      scale_d = 1;
    }
    wgmma_commit();
    wgmma_wait<0>();
    for (int h = 0; h < 2; ++h)
      for (int r = 0; r < 32; ++r) {
        int row, col;
        frag_rc(t, r, row, col);
        o[2 * 64 * 128 + row * 128 + 64 * h + col] = d[h][r];
      }
  }
}

uint64_t g_state = 0x9E3779B97F4A7C15ull;
uint32_t next_u32() {
  g_state = g_state * 6364136223846793005ull + 1442695040888963407ull;
  return (uint32_t)(g_state >> 33);
}
float uniform() { return (next_u32() & 0xFFFFFF) / 16777216.f; }
// odd trials spread the magnitudes over 2^-8 .. 2^8, so the accumulation order shows in the low bits
float sample(int trial) {
  const float v = 2.f * uniform() - 1.f;
  return (trial & 1) ? v * std::ldexp(1.f, (int)(next_u32() % 17) - 8) : v;
}

}  // namespace

int main() {
  const size_t nw = (size_t)kTrials * kMaxTaps * 64 * 64, nx = (size_t)kTrials * kXRows * 64;
  std::vector<__nv_bfloat16> hw(nw), hx(nx);
  for (int tr = 0; tr < kTrials; ++tr) {
    for (size_t i = 0; i < nw / kTrials; ++i) hw[tr * (nw / kTrials) + i] = __float2bfloat16(sample(tr));
    for (size_t i = 0; i < nx / kTrials; ++i) hx[tr * (nx / kTrials) + i] = __float2bfloat16(sample(tr));
  }
  __nv_bfloat16 *dw, *dx;
  float* dout;
  const size_t nout = (size_t)kTrials * 3 * 64 * 128;
  if (cudaMalloc(&dw, nw * 2) || cudaMalloc(&dx, nx * 2) || cudaMalloc(&dout, nout * 4)) { fprintf(stderr, "cudaMalloc failed\n"); return 2; }
  cudaMemcpy(dw, hw.data(), nw * 2, cudaMemcpyHostToDevice);
  cudaMemcpy(dx, hx.data(), nx * 2, cudaMemcpyHostToDevice);
  cudaFuncSetAttribute(probe_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmem);
  std::vector<float> h(nout);
  int bad_total = 0;
  for (int taps : {9, 18}) {
    probe_kernel<<<kTrials, 128, kSmem>>>(dw, dx, taps, dout);
    const cudaError_t err = cudaDeviceSynchronize();
    if (err != cudaSuccess) { fprintf(stderr, "kernel failed: %s\n", cudaGetErrorString(err)); return 2; }
    cudaMemcpy(h.data(), dout, nout * 4, cudaMemcpyDeviceToHost);
    for (int tr = 0; tr < kTrials; ++tr) {
      const float* o = h.data() + (size_t)tr * 3 * 64 * 128;
      int bad128 = 0, bad64 = 0;
      double maxerr = 0, maxref = 0;
      for (int co = 0; co < 64; ++co)
        for (int px = 0; px < 128; ++px) {
          const int i = co * 128 + px;
          bad128 += memcmp(&o[i], &o[64 * 128 + i], 4) != 0;
          bad64 += memcmp(&o[i], &o[2 * 64 * 128 + i], 4) != 0;
          double ref = 0;   // fp64 sanity check of the reference mapping
          for (int tap = 0; tap < taps; ++tap)
            for (int ci = 0; ci < 64; ++ci)
              ref += (double)__bfloat162float(hw[((size_t)tr * kMaxTaps + tap) * 64 * 64 + co * 64 + ci]) *
                     (double)__bfloat162float(hx[((size_t)tr * kXRows + px + tap_shift(tap)) * 64 + ci]);
          maxerr = std::fmax(maxerr, std::fabs(ref - o[i]));
          maxref = std::fmax(maxref, std::fabs(ref));
        }
      printf("k-steps %2d trial %d (%s): n128 vs ref %d / 8192 differ, n64 vs ref %d / 8192 differ, ref max|err| vs fp64 %.3e of max|D| %.3e\n",
             4 * taps, tr, (tr & 1) ? "wide" : "unit", bad128, bad64, maxerr, maxref);
      bad_total += bad128 + bad64;
    }
  }
  printf("%s\n", bad_total == 0 ? "BIT-IDENTICAL" : "DIFFERENT");
  return bad_total == 0 ? 0 : 1;
}
