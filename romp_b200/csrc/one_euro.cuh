// One-Euro smoothing math shared by ROMP's temporal stage (temporal.cu) and BEV's tracker stage (track.cu).
// Restates (fp32, same operation order): LowPassFilter simple_romp/romp/utils.py:203-215, OneEuroFilter :217-246
// (freq 30, dcutoff 1, beta 0.7), and the axis-angle -> matrix step of smooth_global_rot_matrix :188-192 (the
// quaternion form of utils.batch_rodrigues :493-533).
#pragma once

namespace b200romp {

constexpr int kOeCh = 9 + 69 + 16 + 3;       // global-rot matrix | body pose | betas (up to 16) | cam
constexpr int kOeGlob = 0, kOePose = 9, kOeBeta = 78, kOeCam = 94;

__device__ __forceinline__ float oe_alpha(float cutoff, float freq) {     // OneEuroFilter.compute_alpha, utils.py:227-230
  const float te = 1.0f / freq;
  const float tau = 1.0f / (2.0f * 3.14159265358979323846f * cutoff);
  return 1.0f / (1.0f + tau / te);
}

// utils.batch_rodrigues (:493-505) + quat2mat (:507-533) of one axis-angle vector a[3] -> row-major R[9]
__device__ __forceinline__ void oe_rodrigues(const float* a, float* R) {
  const float ex = a[0] + 1e-8f, ey = a[1] + 1e-8f, ez = a[2] + 1e-8f;
  const float nrm = sqrtf(ex * ex + ey * ey + ez * ez);
  const float ux = a[0] / nrm, uy = a[1] / nrm, uz = a[2] / nrm;
  const float h = nrm * 0.5f, c = cosf(h), s = sinf(h);
  float w = c, x = s * ux, y = s * uy, z = s * uz;
  const float qn = sqrtf(w * w + x * x + y * y + z * z);
  w /= qn; x /= qn; y /= qn; z /= qn;
  const float w2 = w * w, x2 = x * x, y2 = y * y, z2 = z * z, wx = w * x, wy = w * y, wz = w * z, xy = x * y, xz = x * z, yz = y * z;
  R[0] = w2 + x2 - y2 - z2; R[1] = 2 * xy - 2 * wz; R[2] = 2 * wy + 2 * xz;
  R[3] = 2 * wz + 2 * xy; R[4] = w2 - x2 + y2 - z2; R[5] = 2 * yz - 2 * wx;
  R[6] = 2 * xz - 2 * wy; R[7] = 2 * wx + 2 * yz; R[8] = w2 - x2 - y2 + z2;
}

// OneEuroFilter.process (:232-246) of one scalar x with the filter state at raw / px / pdx; seen == false: the first
// sample (dx = 0.0, s = value).  Returns the filtered value.
// aliased: the tracked mode of the reference (romp/main.py:152-154, bev/main.py:283-285) hands smooth_results views of
// the output row and then writes the smoothed values into that row; LowPassFilter keeps prev_raw_value = value without
// a copy (:213), so the next dx is taken against the SMOOTHED value.  This holds for pose, betas and cam; the rotation
// matrix is a fresh tensor, and --show_largest rebinds the outputs instead (romp/main.py:133-135), so both keep the raw.
__device__ __forceinline__ float oe_step(float x, float mincut, float freq, bool seen, bool aliased, float* raw, float* px, float* pdx) {
  float y = x;
  if (seen) {
    const float dx = (x - *raw) * freq;                                              // :233-234
    const float ad = oe_alpha(1.0f, freq);
    const float edx = ad * dx + (1.0f - ad) * *pdx;                                  // dx_filter.process, :209-214
    const float cutoff = mincut + 0.7f * fabsf(edx);                                 // :237-242
    const float ax = oe_alpha(cutoff, freq);
    y = ax * x + (1.0f - ax) * *px;                                                  // x_filter.process
    *pdx = edx;
  } else {
    *pdx = 0.0f;
  }
  *raw = aliased ? y : x;
  *px = y;
  return y;
}

}  // namespace b200romp
