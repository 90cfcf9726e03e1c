// Seam S4: projection of joints / vertices into the image and camera translation.
//
// Replaces simple_romp/romp: body_mesh_projection2image post_parser.py:104-114, batch_orth_proj
// utils.py:309-315, convert_proejection_from_input_to_orgimg post_parser.py:81-88,
// convert_cam_to_3d_trans utils.py:303-307 and - for cam_trans - the closed-form weighted least squares
// estimate_translation_np utils.py:347-389 (the reference's fallback for its per-person CPU
// cv2.solvePnPRansac loop, utils.py:391-436), including its validity mask (:404-421).
#include "common.cuh"

namespace b200romp {

// pad_tab (device [B,6] fp32 [top,bottom,left,right,h,w] per frame, may be NULL): person n uses the row of its frame
// batch_ids[n] instead of the shared size / left / top
__global__ void __launch_bounds__(256) project_points_kernel(const float* __restrict__ pts, const float* __restrict__ cam,
                                                             int n_host, const int* __restrict__ d_count, int npts,
                                                             int out_dim, float size, float left, float top,
                                                             const float* __restrict__ pad_tab, const long long* __restrict__ batch_ids,
                                                             float* __restrict__ out) {
  const int n = blockIdx.x;
  const int N = d_count ? min(n_host, *d_count) : n_host;
  if (n >= N) return;
  if (pad_tab) {
    const float* f = pad_tab + batch_ids[n] * 6;
    top = f[0]; left = f[2];
    size = f[4] > f[5] ? f[4] : f[5];                         // post_parser.py:83
  }
  const float s = cam[n * 3 + 0], tx = cam[n * 3 + 1], ty = cam[n * 3 + 2];
  for (int i = blockIdx.y * 256 + threadIdx.x; i < npts; i += gridDim.y * 256) {
    const float* q = pts + ((size_t)n * npts + i) * 3;
    float* o = out + ((size_t)n * npts + i) * out_dim;
    const float x = q[0] * s + tx, y = q[1] * s + ty;         // utils.py:311-312
    o[0] = (x + 1.f) * size / 2.f - left;                     // post_parser.py:84-85
    o[1] = (y + 1.f) * size / 2.f - top;
    if (out_dim == 3) o[2] = (q[2] + 1.f) * size / 2.f;       // :87
  }
}

__global__ void __launch_bounds__(128) cam_trans_kernel(const float* __restrict__ joints, const float* __restrict__ cam,
                                                        int n_host, const int* __restrict__ d_count, float focal,
                                                        float img, float* __restrict__ weak, float* __restrict__ lsq) {
  const int n = blockIdx.x * 128 + threadIdx.x;
  const int N = d_count ? min(n_host, *d_count) : n_host;
  if (n >= N) return;
  const float s = cam[n * 3 + 0], tx = cam[n * 3 + 1], ty = cam[n * 3 + 2];
  if (weak) {                                                 // utils.py:303-307
    weak[n * 3 + 0] = tx / s * 2.f;
    weak[n * 3 + 1] = ty / s * 2.f;
    weak[n * 3 + 2] = 1.f / s * 2.f;
  }
  if (!lsq) return;
  double A[3][3] = {{0, 0, 0}, {0, 0, 0}, {0, 0, 0}}, b[3] = {0, 0, 0};
  const double F = focal, O = img / 2.0;
  int valid = 0;
  for (int i = 0; i < 24; ++i) {
    const float* q = joints + ((size_t)n * 71 + i) * 3;
    const float px = (q[0] * s + tx + 1.f) * 256.f, py = (q[1] * s + ty + 1.f) * 256.f;   // post_parser.py:98
    if (!(py > -2.f) || q[2] == -2.f) continue;               // utils.py:404-408,419
    ++valid;
    const double X = q[0], Y = q[1], Z = q[2];
    const double qx[3] = {F, 0.0, O - px}, qy[3] = {0.0, F, O - py};   // utils.py:374
    const double cx = (px - O) * Z - F * X, cy = (py - O) * Z - F * Y; // :375
    for (int r = 0; r < 3; ++r) {
      for (int c = 0; c < 3; ++c) A[r][c] += qx[r] * qx[c] + qy[r] * qy[c];
      b[r] += qx[r] * cx + qy[r] * cy;
    }
  }
  if (valid < 4) {                                            // utils.py:420-422 INVALID_TRANS
    lsq[n * 3 + 0] = lsq[n * 3 + 1] = lsq[n * 3 + 2] = -1.f;
    return;
  }
  // 3x3 solve (np.linalg.solve, :387) by Gaussian elimination with partial pivoting
  double M[3][4] = {{A[0][0], A[0][1], A[0][2], b[0]}, {A[1][0], A[1][1], A[1][2], b[1]}, {A[2][0], A[2][1], A[2][2], b[2]}};
  for (int c = 0; c < 3; ++c) {
    int piv = c;
    for (int r = c + 1; r < 3; ++r)
      if (fabs(M[r][c]) > fabs(M[piv][c])) piv = r;
    for (int k = 0; k < 4; ++k) { const double t = M[c][k]; M[c][k] = M[piv][k]; M[piv][k] = t; }
    for (int r = c + 1; r < 3; ++r) {
      const double f = M[r][c] / M[c][c];
      for (int k = c; k < 4; ++k) M[r][k] -= f * M[c][k];
    }
  }
  double x[3];
  for (int r = 2; r >= 0; --r) {
    double a = M[r][3];
    for (int k = r + 1; k < 3; ++k) a -= M[r][k] * x[k];
    x[r] = a / M[r][r];
  }
  lsq[n * 3 + 0] = (float)x[0]; lsq[n * 3 + 1] = (float)x[1]; lsq[n * 3 + 2] = (float)x[2];
}

static int project(const float* joints, const float* verts, const float* cam, int n, const int* d_count, const float* offsets6,
                   const long long* batch_ids, const float* pad_table, float* pj2d_org, float* verts_camed_org, float* cam_trans_weak,
                   float* cam_trans_lsq, cudaStream_t stream) {
  float top = 0.f, left = 0.f, size = 0.f;
  if (offsets6) {
    const float h = offsets6[4], w = offsets6[5];
    top = offsets6[0]; left = offsets6[2];
    size = h > w ? h : w;                                    // post_parser.py:83
  }
  if (cam_trans_weak || cam_trans_lsq) {
    cam_trans_kernel<<<(n + 127) / 128, 128, 0, stream>>>(joints, cam, n, d_count, 443.4f, 512.f, cam_trans_weak, cam_trans_lsq);
    B2R_CUDA_OK(cudaGetLastError());
  }
  if (pj2d_org) {
    project_points_kernel<<<dim3(n, 1), 256, 0, stream>>>(joints, cam, n, d_count, 71, 2, size, left, top, pad_table, batch_ids, pj2d_org);
    B2R_CUDA_OK(cudaGetLastError());
  }
  if (verts_camed_org) {
    project_points_kernel<<<dim3(n, 4), 256, 0, stream>>>(verts, cam, n, d_count, 6890, 3, size, left, top, pad_table, batch_ids,
                                                          verts_camed_org);
    B2R_CUDA_OK(cudaGetLastError());
  }
  return B200ROMP_OK;
}

}  // namespace b200romp

using namespace b200romp;

extern "C" int b200romp_project(const float* joints, const float* verts, const float* cam, int n, const int* d_count,
                                const float* offsets6, float* pj2d_org, float* verts_camed_org, float* cam_trans_weak,
                                float* cam_trans_lsq, b200romp_stream stream) {
  B2R_REQUIRE(joints && cam && offsets6 && n > 0, "project: bad arguments");
  B2R_REQUIRE(!verts_camed_org || verts, "project: verts_camed_org requested without verts");
  return project(joints, verts, cam, n, d_count, offsets6, nullptr, nullptr, pj2d_org, verts_camed_org, cam_trans_weak, cam_trans_lsq,
                 (cudaStream_t)stream);
}

extern "C" int b200romp_project_frames(const float* joints, const float* verts, const float* cam, int n, const int* d_count,
                                       const long long* batch_ids, const float* pad_table, float* pj2d_org, float* verts_camed_org,
                                       float* cam_trans_weak, float* cam_trans_lsq, b200romp_stream stream) {
  B2R_REQUIRE(joints && cam && batch_ids && pad_table && n > 0, "project_frames: bad arguments");
  B2R_REQUIRE(!verts_camed_org || verts, "project_frames: verts_camed_org requested without verts");
  return project(joints, verts, cam, n, d_count, nullptr, batch_ids, pad_table, pj2d_org, verts_camed_org, cam_trans_weak,
                 cam_trans_lsq, (cudaStream_t)stream);
}
