// Row a1 / f2: img_preprocess + padding_image (simple_romp/romp/utils.py:16-30) on the GPU:
//   cv2.cvtColor(BGR2RGB) -> centre zero-pad to a square -> cv2.resize(..., (S,S), INTER_CUBIC) -> uint8 [S,S,3]
// in ONE kernel reading the raw BGR image and writing the network's input frame.  One launch covers up to 64 images of
// different sizes (grid z = image), each with its own padded square and scale, and writes each image's pad info to a
// device table the per-frame post stages read.
//
// Bit-exactness target: OpenCV's own 8-bit bicubic resize (modules/imgproc/src/resize.cpp, the algorithm restated from
// its published source; pip wheels additionally carry a closed-source IPP fast path whose results differ from OpenCV's
// own code by +-1 LSB on ~3 % of the pixels and depend on the host CPU):
//   * source coordinate fx = (float)((dx + 0.5) * scale - 0.5), scale = side / S in double; sx = floor(fx); fx -= sx
//   * cubic weights (A = -0.75) evaluated in fp32 in OpenCV's operation order, converted to 11-bit fixed point with
//     round-half-even (saturate_cast<short>(w * 2048)); NO renormalisation of the four taps
//   * horizontal pass in int32 over the 4 taps with replicated borders (index clamp on the padded square)
//   * vertical pass in fp32 exactly like the vectorised VResizeCubic path: t = S3*b3; t = S2*b2 + t; t = S1*b1 + t;
//     t = S0*b0 + t with b_k = beta_k * 2^-22, separate multiply and add roundings (no FMA), round-half-even, saturate.
// The zero padding and the BGR->RGB swap are folded into the tap fetch.
#include "common.cuh"

namespace b200romp {

__device__ __forceinline__ void cubic_taps(int d, double scale, int* s0, int (&w)[4]) {
  float fx = (float)(((double)d + 0.5) * scale - 0.5);
  int s = (int)fx;
  s -= (s > fx);                                   // cvFloor
  fx = __fsub_rn(fx, (float)s);
  const float A = -0.75f;
  const float x1 = __fadd_rn(fx, 1.f);
  float c0 = __fsub_rn(__fmul_rn(__fadd_rn(__fmul_rn(__fsub_rn(__fmul_rn(A, x1), __fmul_rn(5.f, A)), x1), __fmul_rn(8.f, A)), x1), __fmul_rn(4.f, A));
  float c1 = __fadd_rn(__fmul_rn(__fmul_rn(__fsub_rn(__fmul_rn(__fadd_rn(A, 2.f), fx), __fadd_rn(A, 3.f)), fx), fx), 1.f);
  const float xm = __fsub_rn(1.f, fx);
  float c2 = __fadd_rn(__fmul_rn(__fmul_rn(__fsub_rn(__fmul_rn(__fadd_rn(A, 2.f), xm), __fadd_rn(A, 3.f)), xm), xm), 1.f);
  float c3 = __fsub_rn(__fsub_rn(__fsub_rn(1.f, c0), c1), c2);
  w[0] = __float2int_rn(__fmul_rn(c0, 2048.f));
  w[1] = __float2int_rn(__fmul_rn(c1, 2048.f));
  w[2] = __float2int_rn(__fmul_rn(c2, 2048.f));
  w[3] = __float2int_rn(__fmul_rn(c3, 2048.f));
  *s0 = s;
}

// One image of a batch: device pointer, size, row stride, padded square and its resize scale (host-computed, so the
// arithmetic is that of the single-image case).  A batch travels to the kernel as a launch parameter (no descriptor table
// in device memory, no H2D copy).
struct PreprocImage {
  const unsigned char* img;
  int h, w, row_stride, side, top, left;
  double scale;
};
constexpr int kPreprocBatch = 64;     // images per launch: 64 x 40 B of descriptors stay well inside the 4 KB parameter space
struct PreprocBatch { PreprocImage im[kPreprocBatch]; };

// thread = one output pixel (3 channels) of image blockIdx.z; pad_tab (device [n,6] fp32, may be NULL) receives each
// image's [top, bottom, left, right, h, w] (utils.py:24)
__global__ void __launch_bounds__(256) preprocess_bgr_kernel(const __grid_constant__ PreprocBatch batch, int S,
                                                             unsigned char* __restrict__ out, float* __restrict__ pad_tab) {
  const PreprocImage& im = batch.im[blockIdx.z];
  const int dx = blockIdx.x * blockDim.x + threadIdx.x, dy = blockIdx.y;
  if (pad_tab && dx == 0 && dy == 0) {
    float* p = pad_tab + (size_t)blockIdx.z * 6;
    p[0] = (float)im.top; p[1] = (float)(im.top + im.h); p[2] = (float)im.left; p[3] = (float)(im.left + im.w);
    p[4] = (float)im.h; p[5] = (float)im.w;
  }
  if (dx >= S) return;
  const unsigned char* __restrict__ img = im.img;
  const int h = im.h, w = im.w, row_stride = im.row_stride, side = im.side, top = im.top, left = im.left;
  int sx, sy, ax[4], ay[4];
  cubic_taps(dx, im.scale, &sx, ax);
  cubic_taps(dy, im.scale, &sy, ay);
  int rows[4][3];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int py = min(max(sy + k - 1, 0), side - 1) - top;          // replicate border of the padded square, then un-pad
    int v0 = 0, v1 = 0, v2 = 0;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int px = min(max(sx + j - 1, 0), side - 1) - left;
      if ((unsigned)py < (unsigned)h && (unsigned)px < (unsigned)w) {
        const unsigned char* p = img + (size_t)py * row_stride + (size_t)px * 3;
        v0 += (int)p[2] * ax[j];                                        // RGB <- BGR
        v1 += (int)p[1] * ax[j];
        v2 += (int)p[0] * ax[j];
      }
    }
    rows[k][0] = v0; rows[k][1] = v1; rows[k][2] = v2;
  }
  const float sc = 1.f / (2048.f * 2048.f);
  const float b0 = __fmul_rn((float)ay[0], sc), b1 = __fmul_rn((float)ay[1], sc), b2 = __fmul_rn((float)ay[2], sc), b3 = __fmul_rn((float)ay[3], sc);
  unsigned char* o = out + (((size_t)blockIdx.z * S + dy) * S + dx) * 3;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    float t = __fmul_rn((float)rows[3][c], b3);
    t = __fadd_rn(__fmul_rn((float)rows[2][c], b2), t);
    t = __fadd_rn(__fmul_rn((float)rows[1][c], b1), t);
    t = __fadd_rn(__fmul_rn((float)rows[0][c], b0), t);
    o[c] = (unsigned char)min(max(__float2int_rn(t), 0), 255);
  }
}

static PreprocImage preproc_image(const unsigned char* img, int h, int w, int row_stride, int out_size) {
  PreprocImage im;
  im.img = img; im.h = h; im.w = w; im.row_stride = row_stride;
  im.side = h > w ? h : w;
  im.top = (im.side - h) / 2; im.left = (im.side - w) / 2;
  im.scale = (double)im.side / (double)out_size;
  return im;
}

}  // namespace b200romp

using namespace b200romp;

extern "C" int b200romp_preprocess_bgr_batch(const unsigned char* const* imgs_bgr, const int* h, const int* w, const int* row_stride_bytes,
                                             int n, int out_size, unsigned char* out_rgb, float* pad_table, b200romp_stream stream) {
  B2R_REQUIRE(imgs_bgr && h && w && row_stride_bytes && n > 0 && out_size > 0 && out_rgb, "preprocess_bgr_batch: bad arguments");
  for (int i = 0; i < n; ++i)
    B2R_REQUIRE(imgs_bgr[i] && h[i] > 0 && w[i] > 0 && row_stride_bytes[i] >= 3 * w[i], "preprocess_bgr_batch: bad image");
  const size_t frame = (size_t)out_size * out_size * 3;
  for (int i0 = 0; i0 < n; i0 += kPreprocBatch) {
    const int nb = n - i0 < kPreprocBatch ? n - i0 : kPreprocBatch;
    PreprocBatch batch;
    for (int i = 0; i < nb; ++i) batch.im[i] = preproc_image(imgs_bgr[i0 + i], h[i0 + i], w[i0 + i], row_stride_bytes[i0 + i], out_size);
    dim3 grid((out_size + 255) / 256, out_size, nb);
    preprocess_bgr_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(batch, out_size, out_rgb + i0 * frame,
                                                                 pad_table ? pad_table + (size_t)i0 * 6 : nullptr);
    B2R_CUDA_OK(cudaGetLastError());
  }
  return B200ROMP_OK;
}

extern "C" int b200romp_preprocess_bgr(const unsigned char* img_bgr, int h, int w, int row_stride_bytes, int out_size,
                                       unsigned char* out_rgb, float* pad_info6, b200romp_stream stream) {
  B2R_REQUIRE(img_bgr && out_rgb && h > 0 && w > 0 && row_stride_bytes >= 3 * w && out_size > 0, "preprocess_bgr: bad arguments");
  if (pad_info6) {                     // utils.py:24: [top, bottom, left, right, h, w]
    const PreprocImage im = preproc_image(img_bgr, h, w, row_stride_bytes, out_size);
    pad_info6[0] = (float)im.top; pad_info6[1] = (float)(im.top + h); pad_info6[2] = (float)im.left; pad_info6[3] = (float)(im.left + w);
    pad_info6[4] = (float)h; pad_info6[5] = (float)w;
  }
  return b200romp_preprocess_bgr_batch(&img_bgr, &h, &w, &row_stride_bytes, 1, out_size, out_rgb, nullptr, stream);
}
