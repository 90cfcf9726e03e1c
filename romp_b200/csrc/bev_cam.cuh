// BEV's camera -> translation conversion, shared by the long-image merge (bev.cu) and the tracker stage (track.cu).
#pragma once

namespace b200romp {

constexpr float kTanFov = 0.57735026919f;   // tan(radians(60/2)), bev/post_parser.py:109

// denormalize_cam_params_to_trans (bev/post_parser.py:114-128) of one cam [s, y, x], rounded op by op like the torch ops
__device__ __forceinline__ void bev_cam_trans_rn(const float* cam, float* trans) {
  const float depth = __fdiv_rn(1.f, __fadd_rn(__fmul_rn(cam[0], kTanFov), 1e-3f));
  trans[0] = __fmul_rn(__fmul_rn(cam[2], depth), kTanFov);
  trans[1] = __fmul_rn(__fmul_rn(cam[1], depth), kTanFov);
  trans[2] = depth;
}

}  // namespace b200romp
