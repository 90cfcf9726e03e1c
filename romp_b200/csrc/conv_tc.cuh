// wgmma implicit-GEMM convolution engine (interface).  Implementation: conv_tc.cu
#pragma once
#include <cuda.h>

#include <string>
#include <vector>

#include "common.cuh"

namespace b200romp {

struct S2Maps {
  CUtensorMap m[4];
};

struct TcConvPlan {
  int kind = 0;                 // kernel family: 10 = 1x1, 30 = 3x3, 31 = 3x3 with the weights as the wgmma A operand
                                // (conv_tc.cu SWAP), 34 = 3x3 with streamed weights as A (conv_tc_stream_kernel),
                                // 32 = 3x3 stride 2, 33 = u8 stem, 13 = conv1d,
                                // 60 = fused 3x3 BasicBlock (conv_block_tc.cu), 70 = fused Bottleneck
                                // (conv_bottleneck_tc.cu); 0 = none
  int cin = 0, cout = 0, nt = 0;  // channels, output channels per CTA
  int eb = 2;                   // operand element bytes: 2 = bf16, 4 = fp32 storage consumed as TF32
  int grid_x = 0, grid_y = 0, stages = 0;
  int smem_bytes = 0;
  void* d_wpack = nullptr;      // weights pre-arranged as the shared-memory image (bf16, swizzled)
  CUtensorMap tmap_in;          // the input tensor
  S2Maps tmap_s2;               // stride-2: one map per input parity (ph,pw)
  // bit (tap * 2 + half) = 0 skips the MMAs of that channel half of that tap (all-zero weights of a pixel-pair folded
  // conv, see net.cu fold_pixel_pairs)
  unsigned kmask = 0xFFFFFFFFu;
  const void* encoded_in = nullptr;   // conv1d engine: input pointer / batch the tensor map was encoded for
  int encoded_batch = 0;
  void* d_wpack2 = nullptr;           // fused block / Bottleneck: conv2's weight image (d_wpack holds conv1's)
  void* d_wpack3 = nullptr;           // fused Bottleneck: conv3's weight image
  const float* d_bias1 = nullptr;     // fused block / Bottleneck: conv1's bias [64] (the last conv's is ConvParams::bias)
  const float* d_bias2 = nullptr;     // fused Bottleneck: conv2's bias [64]
  int fold = 0;                       // set before prepare: runs on the pixel-pair view (net.cu fold_pixel_pairs)
  std::string describe() const;
};

// *_supported: no allocation or CUDA call, a null pointer is a tensor bound later.  A prepare, on a supported shape only,
// packs weights and builds the plan; device allocations are appended to `allocs`.
bool tc_conv_supported(const ConvParams& p, int ksize, int stride);   // includes the shared-memory fit of the weights
int tc_conv_prepare(const ConvParams& p, int ksize, int stride, const float* w_oihw, int sm_count, TcConvPlan* plan,
                    std::vector<void*>* allocs);
int tc_conv_launch(const TcConvPlan& plan, const ConvParams& p, cudaStream_t stream);
// Conv1d (ksize code 13 = 1x3 along W) engine with streamed weights (conv1d_tc.cu): BEV's bird's-eye-view stack
bool tc_conv1d_supported(const ConvParams& p);
int tc_conv1d_prepare(const ConvParams& p, const float* w_oi3, int sm_count, TcConvPlan* plan, std::vector<void*>* allocs);
int tc_conv1d_launch(TcConvPlan& plan, const ConvParams& p, cudaStream_t stream);
// stem engine (conv_stem_tc.cu): 3->64 3x3 stride-2 conv on raw u8 frames with the input normalisation folded in
bool tc_stem_supported(const ConvParams& p, int ksize, int stride);
int tc_stem_prepare(const ConvParams& p, const float* w_oihw, int sm_count, TcConvPlan* plan, std::vector<void*>* allocs);
int tc_stem_launch(const TcConvPlan& plan, const ConvParams& p, cudaStream_t stream);
// fused BasicBlock engine (conv_block_tc.cu): y = relu(conv2(relu(conv1(x) + b1)) + b2 + x), 3x3 stride 1, 64 -> 64 -> 64
// bf16 NHWC.  `p` describes the block as one op: input and residual x (the same channel slice), output y, bias b2; when
// plan->fold the weights are already the pixel-pair folded ones and `p` the pixel-pair view.
bool tc_block_supported(const ConvParams& p, bool fold);
int tc_block_prepare(const ConvParams& p, const float* w1_oihw, const float* b1, const float* w2_oihw, int sm_count,
                     TcConvPlan* plan, std::vector<void*>* allocs);
int tc_block_launch(const TcConvPlan& plan, const ConvParams& p, cudaStream_t stream);
// fused Bottleneck engine (conv_bottleneck_tc.cu): y = relu(W3 relu(W2 * relu(W1 x + b1) + b2) + b3 + x) with 1x1 256 -> 64,
// 3x3 stride-1 64 -> 64 and 1x1 64 -> 256 convs, bf16 NHWC.  `p` describes the block as one op: input and residual x (the
// same 256-channel slice), output y, bias b3.
// `BottleneckMids` are set when other ops of the net also read t1 or t2 (whole 64-channel slices of bf16 NHWC tensors at
// the block's resolution); the kernel then writes them as well.
struct BottleneckMids {
  __nv_bfloat16* t1 = nullptr;
  __nv_bfloat16* t2 = nullptr;
  int t1_C = 0, t2_C = 0;
};
bool tc_bottleneck_supported(const ConvParams& p);
int tc_bottleneck_prepare(const ConvParams& p, const float* w1_oihw, const float* b1, const float* w2_oihw, const float* b2,
                          const float* w3_oihw, int sm_count, TcConvPlan* plan, std::vector<void*>* allocs);
int tc_bottleneck_launch(const TcConvPlan& plan, const ConvParams& p, const BottleneckMids& mids, cudaStream_t stream);

}  // namespace b200romp
