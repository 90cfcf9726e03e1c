// Row f4: the temporal stage of ROMP.forward (simple_romp/romp/main.py:117-157, --temporal_optimize): One-Euro smoothing
// of (smpl_thetas, smpl_betas, cam) per tracked person between the parse (seam S2) and the SMPL forward (seam S3),
// as a streaming device stage: filter state lives in device memory (one slot per track), one kernel per frame batch.
//
// Restates (fp32, same operation order): LowPassFilter utils.py:203-215, OneEuroFilter :217-246 (freq 30, dcutoff 1,
// beta 0.7), create_OneEuroFilter :258-259 (mincutoff: thetas = global_rot = smooth_coeff, cam 1.6, betas 0.6),
// smooth_results :262-270, smooth_global_rot_matrix :188-192 (axis-angle -> matrix via the quaternion form of
// utils.batch_rodrigues :493-533, filter the 9 entries, rotation_matrix_to_angle_axis :535-552 of the filtered matrix).
// The track association itself (norfair in the reference, a third-party tracker that is not part of the repository) is
// host logic in romp_b200/temporal.py; this file only needs the slot index of every person.
#include "common.cuh"
#include "rot6d.cuh"
#include "one_euro.cuh"

namespace b200romp {

struct OeState {
  float* prev_raw;      // [slots][kOeCh]  LowPassFilter.prev_raw_value of the x filter
  float* prev_x;        // [slots][kOeCh]  prev_filtered_value of the x filter
  float* prev_dx;       // [slots][kOeCh]  prev_filtered_value of the dx filter
  int* seen;            // [slots] 0 = the next sample initialises the filters
};

// block = one person, thread = one filtered scalar
__global__ void __launch_bounds__(128) one_euro_kernel(OeState st, const int* __restrict__ slot, int n_host, const int* __restrict__ d_count,
                                                       float* __restrict__ thetas, float* __restrict__ betas, int betas_stride, int n_betas,
                                                       float* __restrict__ cam, float smooth_coeff, float freq) {
  const int i = blockIdx.x;
  const int N = d_count ? min(n_host, *d_count) : n_host;
  if (i >= N) return;
  const int sl = slot[i];
  if (sl < 0) return;
  __shared__ float s_R[9];
  const int t = threadIdx.x;
  if (t == 0) oe_rodrigues(thetas + (size_t)i * 72, s_R);      // utils.batch_rodrigues (:493-505) + quat2mat (:507-533)
  __syncthreads();
  float x = 0.f, mincut = smooth_coeff;
  bool active = true;
  if (t < kOePose) x = s_R[t];
  else if (t < kOeBeta) x = thetas[(size_t)i * 72 + 3 + (t - kOePose)];
  else if (t < kOeCam) { active = (t - kOeBeta) < n_betas; if (active) x = betas[(size_t)i * betas_stride + (t - kOeBeta)]; mincut = 0.6f; }
  else if (t < kOeCh) { x = cam[(size_t)i * 3 + (t - kOeCam)]; mincut = 1.6f; }
  else active = false;
  float y = x;
  if (active) {
    const size_t o = (size_t)sl * kOeCh + t;
    y = oe_step(x, mincut, freq, st.seen[sl] != 0, &st.prev_raw[o], &st.prev_x[o], &st.prev_dx[o]);
  }
  if (t < kOePose) s_R[t] = y;
  else if (t < kOeBeta) thetas[(size_t)i * 72 + 3 + (t - kOePose)] = y;
  else if (t < kOeCam) { if (active) betas[(size_t)i * betas_stride + (t - kOeBeta)] = y; }
  else if (t < kOeCh) cam[(size_t)i * 3 + (t - kOeCam)] = y;
  __syncthreads();
  if (t == 0) {
    float aa[3];
    rotmat_to_aa(s_R, aa);                                                             // :191
    thetas[(size_t)i * 72 + 0] = aa[0]; thetas[(size_t)i * 72 + 1] = aa[1]; thetas[(size_t)i * 72 + 2] = aa[2];
    st.seen[sl] = 1;
  }
}

}  // namespace b200romp

using namespace b200romp;

struct b200romp_tracks {
  int device = 0, slots = 0;
  OeState st{};
};

extern "C" {

b200romp_tracks* b200romp_tracks_create(int device, int max_tracks) {
  if (max_tracks <= 0 || cudaSetDevice(device) != cudaSuccess) {
    set_error("tracks_create: bad arguments / no CUDA device");
    return nullptr;
  }
  b200romp_tracks* t = new b200romp_tracks();
  t->device = device; t->slots = max_tracks;
  const size_t nf = (size_t)max_tracks * kOeCh * sizeof(float);
  if (cudaMalloc(&t->st.prev_raw, nf) != cudaSuccess || cudaMalloc(&t->st.prev_x, nf) != cudaSuccess ||
      cudaMalloc(&t->st.prev_dx, nf) != cudaSuccess || cudaMalloc(&t->st.seen, max_tracks * sizeof(int)) != cudaSuccess ||
      cudaMemset(t->st.seen, 0, max_tracks * sizeof(int)) != cudaSuccess) {
    set_error("tracks_create: allocation failed");
    delete t;
    return nullptr;
  }
  return t;
}

void b200romp_tracks_destroy(b200romp_tracks* t) {
  if (!t) return;
  cudaSetDevice(t->device);
  cudaFree(t->st.prev_raw); cudaFree(t->st.prev_x); cudaFree(t->st.prev_dx); cudaFree(t->st.seen);
  delete t;
}

int b200romp_tracks_reset(b200romp_tracks* t, int slot, b200romp_stream stream) {
  B2R_REQUIRE(t && slot >= -1 && slot < t->slots, "tracks_reset: bad slot");
  B2R_CUDA_OK(cudaSetDevice(t->device));
  if (slot < 0) B2R_CUDA_OK(cudaMemsetAsync(t->st.seen, 0, t->slots * sizeof(int), (cudaStream_t)stream));
  else B2R_CUDA_OK(cudaMemsetAsync(t->st.seen + slot, 0, sizeof(int), (cudaStream_t)stream));
  return B200ROMP_OK;
}

int b200romp_one_euro_smooth(b200romp_tracks* t, const int* slot, int n, const int* d_count, float* thetas, float* betas,
                             int betas_stride, int n_betas, float* cam, float smooth_coeff, float freq, b200romp_stream stream) {
  B2R_REQUIRE(t && slot && thetas && betas && cam && n > 0 && n_betas > 0 && n_betas <= 16 && betas_stride >= n_betas, "one_euro_smooth: bad arguments");
  B2R_CUDA_OK(cudaSetDevice(t->device));
  one_euro_kernel<<<n, 128, 0, (cudaStream_t)stream>>>(t->st, slot, n, d_count, thetas, betas, betas_stride, n_betas, cam, smooth_coeff, freq);
  B2R_CUDA_OK(cudaGetLastError());
  return B200ROMP_OK;
}

}  // extern "C"
