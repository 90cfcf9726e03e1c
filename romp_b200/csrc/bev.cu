// BEV-specific stages of the hot path (workload cfg3): everything of simple_romp/bev/model.py and
// bev/post_parser.py that is not a 2-D / 1-D convolution (those run on the conv-graph engines).
//
//   bev_bv_input      : torch.cat([center_fv, cam_offset, img_feats],1).view(B,-1,128)           bev/model.py:190
//   bev_center3d      : outer product fv x bv + BasicBlock_3D(1->1) refiner                       :195-196,206 (+:52-75)
//   bev_parse3d       : CenterMap3D.parse_3dcentermap (5x5x5 max-pool NMS, top-64, threshold)     bev/post_parser.py:44-66
//   bev_regress       : cam_maps_3d sampled at the detections - evaluated LAZILY: the BasicBlock_3D(3->3) refiner is
//                       computed only on the 5^3 neighbourhood of each detection instead of materialising the
//                       [B,3,64,128,128] volume (12.6 MB/frame) - then anchor arg-min, feature sampling + position
//                       embedding and the 128-512-512-143 MLP                                     bev/model.py:209-213,217-230,242
//   bev_unpack        : pack_params_dict (11 betas) + denormalize_cam_params_to_trans             bev/post_parser.py:240-253,114-128
//   bev_merge_smil    : SMPLA_parser's baby/adult split (betas[:,10] > 0.8)                       :255-278
//   bev_project       : perspective_projection (f=443.4) + convert to original-image pixels       :68-107,129-152
//   bev_postfilter    : suppressing_redundant_prediction_via_projection + remove_outlier, applied per frame
//                       (the reference assumes one frame)                                         :167-222
// All fp32, one host sync per batch (the final person count).
#include <math_constants.h>

#include <vector>

#include "common.cuh"
#include "rot6d.cuh"
#include "bev_cam.cuh"

namespace b200romp {

constexpr int kD = 64, kS = 128, kVol = kD * kS * kS;
constexpr int kCandCap = 4096;          // local maxima above threshold kept per frame before the top-64 sort
constexpr int kMaxP = 64;

struct BevDev {
  const float* center_ref;   // [56]  w1[27] b1 w2[27] b2   (BatchNorm3d folded)
  const float* cam_ref;      // [492] w1[3][3][27] b1[3] w2[3][3][27] b2[3]
  const float* coordmap;     // [64][128][128][3]
  const float* anchors;      // [64]
  const float* embed;        // [128][128]
  const float *w0t, *b0, *w1t, *b1, *w2t, *b2;   // MLP, weights transposed to [in][out]
};

// ---------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) bev_bv_input_kernel(const float* __restrict__ maps_fv, const void* __restrict__ feats,
                                                           int feats_dtype, int feats_C, int B, void* __restrict__ out, int out_dtype) {
  const size_t idx = (size_t)blockIdx.x * 256 + threadIdx.x;
  if (idx >= (size_t)B * kS * 2560) return;
  const int ch = idx % 2560, w = (idx / 2560) % kS, b = idx / ((size_t)2560 * kS);
  const int c = ch / kS, h = ch % kS;
  float v;
  if (c < 4) v = maps_fv[(((size_t)b * 4 + c) * kS + h) * kS + w];
  else v = load_as_float(feats, (((size_t)b * kS + h) * kS + w) * feats_C + (c - 4), feats_dtype);
  store_from_float(out, idx, out_dtype, v);
}

// center_map_3d = fv (x) bv, refined by BasicBlock_3D(1->1).  stage 1: t1 = relu(bn1(conv1(cm))); stage 2: bn2(conv2(t1)) + cm
__device__ __forceinline__ float cm_at(const float* cfv, const void* bv, int bv_dtype, int b, int d, int h, int w) {
  return cfv[((size_t)b * 4 * kS + h) * kS + w] * load_as_float(bv, ((size_t)b * kS + w) * kS + d, bv_dtype);
}

__global__ void __launch_bounds__(256) bev_center3d_kernel(const float* __restrict__ maps_fv, const void* __restrict__ bv,
                                                           int bv_dtype, BevDev m, int B, const float* __restrict__ t1,
                                                           float* __restrict__ out, int stage) {
  const size_t idx = (size_t)blockIdx.x * 256 + threadIdx.x;
  if (idx >= (size_t)B * kVol) return;
  const int w = idx % kS, h = (idx / kS) % kS, d = (idx / (kS * kS)) % kD, b = idx / kVol;
  const float* wgt = m.center_ref + (stage == 1 ? 0 : 28);
  float acc = wgt[27];
#pragma unroll
  for (int dz = -1; dz <= 1; ++dz)
#pragma unroll
    for (int dy = -1; dy <= 1; ++dy)
#pragma unroll
      for (int dx = -1; dx <= 1; ++dx) {
        const int zz = d + dz, yy = h + dy, xx = w + dx;
        if (zz < 0 || zz >= kD || yy < 0 || yy >= kS || xx < 0 || xx >= kS) continue;
        const float x = stage == 1 ? cm_at(maps_fv, bv, bv_dtype, b, zz, yy, xx)
                                   : t1[(((size_t)b * kD + zz) * kS + yy) * kS + xx];
        acc = fmaf(wgt[(dz + 1) * 9 + (dy + 1) * 3 + (dx + 1)], x, acc);
      }
  out[idx] = stage == 1 ? fmaxf(acc, 0.f) : acc + cm_at(maps_fv, bv, bv_dtype, b, d, h, w);
}

// Fused version of the two stages above (round 2): one kernel, the intermediate t1 never leaves shared memory, and stage 1
// uses the rank-1 structure of its input: cm[d,h,w] = fv[h,w] * bv[w,d], so
//     conv1(cm)[d,h,w] = sum_{a,c} bv[w+c, d+a] * G[a,c][h, w+c],   G[a,c][h,x] = sum_b k1[a,b,c] * fv[h+b, x]
// (9 FMA per voxel instead of 27; G is 9 planes of the block's 10 x 36 footprint).  Stage 2 is the full 27-tap stencil on the
// shared-memory t1 tile with a sliding window along d.  Block = 8 (d) x 8 (h) x 32 (w) outputs, 256 threads.
// FLOPs per output: 9 * (10*10*34)/(8*8*32) + 27 = 42 (was 54), global traffic: one fp32 store per voxel (was 3 accesses).
constexpr int kTD = 8, kTH = 8, kTW = 32;
__global__ void __launch_bounds__(256) bev_center3d_fused_kernel(const float* __restrict__ maps_fv, const void* __restrict__ bv,
                                                                 int bv_dtype, BevDev m, float* __restrict__ out) {
  __shared__ float s_fv[kTH + 4][kTW + 4];            // fv rows h0-2 .. h0+9, cols w0-2 .. w0+33 (zero outside the map)
  __shared__ float s_bv[kTW + 4][kTD + 4];            // bv[w][d] cols w0-2.., depth d0-2 .. d0+9 (zero outside)
  __shared__ float s_G[9][kTH + 2][kTW + 4];          // G[a*3+c][h0-1 .. h0+8][w0-2 .. w0+33]
  __shared__ float s_t1[kTD + 2][kTH + 2][kTW + 2];   // relu(conv1 + b1) on the halo tile, zero outside the volume
  const int b = blockIdx.z;
  const int w0 = (blockIdx.x % (kS / kTW)) * kTW, h0 = (blockIdx.x / (kS / kTW)) * kTH, d0 = blockIdx.y * kTD;
  const int tid = threadIdx.x;
  const float* cfv = maps_fv + (size_t)b * 4 * kS * kS;            // channel 0 = center_maps_fv
  for (int i = tid; i < (kTH + 4) * (kTW + 4); i += 256) {
    const int r = i / (kTW + 4), c = i % (kTW + 4), h = h0 - 2 + r, w = w0 - 2 + c;
    s_fv[r][c] = (h >= 0 && h < kS && w >= 0 && w < kS) ? cfv[(size_t)h * kS + w] : 0.f;
  }
  for (int i = tid; i < (kTW + 4) * (kTD + 4); i += 256) {
    const int c = i / (kTD + 4), r = i % (kTD + 4), w = w0 - 2 + c, d = d0 - 2 + r;
    s_bv[c][r] = (w >= 0 && w < kS && d >= 0 && d < kD) ? load_as_float(bv, ((size_t)b * kS + w) * kS + d, bv_dtype) : 0.f;
  }
  __syncthreads();
  const float* k1 = m.center_ref;                       // [27] then b1
  for (int i = tid; i < 9 * (kTH + 2) * (kTW + 4); i += 256) {
    const int x = i % (kTW + 4), r = (i / (kTW + 4)) % (kTH + 2), ac = i / ((kTW + 4) * (kTH + 2));
    const int a = ac / 3, c = ac % 3;
    // G[a,c][h0-1+r][w0-2+x] = sum_b k1[a][b][c] * fv[h0-1+r + (b-1)][.]  (s_fv row index = r + b)
    s_G[ac][r][x] = k1[a * 9 + 0 * 3 + c] * s_fv[r + 0][x] + k1[a * 9 + 1 * 3 + c] * s_fv[r + 1][x] + k1[a * 9 + 2 * 3 + c] * s_fv[r + 2][x];
  }
  __syncthreads();
  const float b1 = k1[27];
  for (int i = tid; i < (kTH + 2) * (kTW + 2); i += 256) {      // one (h, w) column of the t1 halo tile per iteration
    const int wl = i % (kTW + 2), hl = i / (kTW + 2);            // t1 position (h0-1+hl, w0-1+wl); s_G / s_bv column index = wl + 1 + (c-1)
    const int h = h0 - 1 + hl, w = w0 - 1 + wl;
    const bool inside_hw = h >= 0 && h < kS && w >= 0 && w < kS;
    float g[9];
#pragma unroll
    for (int ac = 0; ac < 9; ++ac) g[ac] = s_G[ac][hl][wl + (ac % 3)];
#pragma unroll
    for (int dl = 0; dl < kTD + 2; ++dl) {                       // t1 depth d0-1+dl; s_bv depth index = dl + 1 + (a-1)
      float acc = b1;
#pragma unroll
      for (int a = 0; a < 3; ++a)
#pragma unroll
        for (int c = 0; c < 3; ++c) acc = fmaf(s_bv[wl + c][dl + a], g[a * 3 + c], acc);
      const int d = d0 - 1 + dl;
      s_t1[dl][hl][wl] = (inside_hw && d >= 0 && d < kD) ? fmaxf(acc, 0.f) : 0.f;
    }
  }
  __syncthreads();
  const float* k2 = m.center_ref + 28;                  // [27] then b2
  float wk[27];
#pragma unroll
  for (int i = 0; i < 27; ++i) wk[i] = k2[i];
  const float b2 = k2[27];
  const int wl = tid % kTW, hl = tid / kTW;             // output (h0+hl, w0+wl), all kTD depths
  float p0[9], p1[9], p2[9];                            // t1 planes d-1, d, d+1 (3x3 in h, w)
#pragma unroll
  for (int j = 0; j < 9; ++j) { p0[j] = s_t1[0][hl + j / 3][wl + j % 3]; p1[j] = s_t1[1][hl + j / 3][wl + j % 3]; }
  const float fvv = s_fv[hl + 2][wl + 2];
#pragma unroll
  for (int dl = 0; dl < kTD; ++dl) {
#pragma unroll
    for (int j = 0; j < 9; ++j) p2[j] = s_t1[dl + 2][hl + j / 3][wl + j % 3];
    float acc = b2;
#pragma unroll
    for (int j = 0; j < 9; ++j) acc = fmaf(wk[j], p0[j], acc);
#pragma unroll
    for (int j = 0; j < 9; ++j) acc = fmaf(wk[9 + j], p1[j], acc);
#pragma unroll
    for (int j = 0; j < 9; ++j) acc = fmaf(wk[18 + j], p2[j], acc);
    const float cm = fvv * s_bv[wl + 2][dl + 2];
    out[(((size_t)b * kD + d0 + dl) * kS + h0 + hl) * kS + w0 + wl] = acc + cm;
#pragma unroll
    for (int j = 0; j < 9; ++j) { p0[j] = p1[j]; p1[j] = p2[j]; }
  }
}

// ---------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) bev_nms3d_kernel(const float* __restrict__ c3d, int B, float thresh,
                                                        int* __restrict__ cand_count, int* __restrict__ cand_idx,
                                                        float* __restrict__ cand_val) {
  const size_t idx = (size_t)blockIdx.x * 256 + threadIdx.x;
  if (idx >= (size_t)B * kVol) return;
  const float v = c3d[idx];
  if (!(v > thresh)) return;                       // det * (maxpool == det) > thresh  <=>  det > thresh and det is a maximum
  const int vox = idx % kVol, b = idx / kVol;
  const int x = vox % kS, y = (vox / kS) % kS, z = vox / (kS * kS);
  const float* base = c3d + (size_t)b * kVol;
  for (int dz = -2; dz <= 2; ++dz) {
    const int zz = z + dz;
    if (zz < 0 || zz >= kD) continue;
    for (int dy = -2; dy <= 2; ++dy) {
      const int yy = y + dy;
      if (yy < 0 || yy >= kS) continue;
      for (int dx = -2; dx <= 2; ++dx) {
        const int xx = x + dx;
        if (xx < 0 || xx >= kS) continue;
        if (base[((size_t)zz * kS + yy) * kS + xx] > v) return;
      }
    }
  }
  const int slot = atomicAdd(&cand_count[b], 1);
  if (slot < kCandCap) {
    cand_idx[(size_t)b * kCandCap + slot] = vox;
    cand_val[(size_t)b * kCandCap + slot] = v;
  }
}

__device__ __forceinline__ bool before3(float ka, int ia, float kb, int ib) { return (ka > kb) || (ka == kb && ia < ib); }

__global__ void __launch_bounds__(1024) bev_top64_kernel(const int* __restrict__ cand_count, const int* __restrict__ cand_idx,
                                                         const float* __restrict__ cand_val, int* __restrict__ counts,
                                                         int* __restrict__ top_idx, float* __restrict__ top_val) {
  __shared__ float s_key[kCandCap];
  __shared__ int s_idx[kCandCap];
  const int b = blockIdx.x, tid = threadIdx.x;
  const int n = min(cand_count[b], kCandCap);
  for (int i = tid; i < kCandCap; i += 1024) {
    s_key[i] = i < n ? cand_val[(size_t)b * kCandCap + i] : -CUDART_INF_F;
    s_idx[i] = i < n ? cand_idx[(size_t)b * kCandCap + i] : 0x7fffffff;
  }
  __syncthreads();
  for (int k = 2; k <= kCandCap; k <<= 1)
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int t = tid; t < kCandCap / 2; t += 1024) {
        const int lo = ((t / j) * 2 * j) + (t % j), hi = lo + j;
        const bool up = ((lo & k) == 0);
        const float ka = s_key[lo], kb = s_key[hi];
        const int ia = s_idx[lo], ib = s_idx[hi];
        if (before3(ka, ia, kb, ib) != up) {
          s_key[lo] = kb; s_key[hi] = ka; s_idx[lo] = ib; s_idx[hi] = ia;
        }
      }
      __syncthreads();
    }
  if (tid < kMaxP) {
    top_idx[b * kMaxP + tid] = s_idx[tid];
    top_val[b * kMaxP + tid] = s_key[tid];
  }
  if (tid == 0) counts[b] = min(n, kMaxP);
}

__global__ void __launch_bounds__(64) bev_emit_kernel(int B, int capacity, const int* __restrict__ counts,
                                                      const int* __restrict__ top_idx, const float* __restrict__ top_val,
                                                      int* __restrict__ d_count, long long* __restrict__ batch_ids,
                                                      long long* __restrict__ czyx, float* __restrict__ conf) {
  const int b = blockIdx.x, tid = threadIdx.x;
  __shared__ int s_off;
  if (tid == 0) {
    int o = 0;
    for (int i = 0; i < b; ++i) o += counts[i];
    s_off = o;
    if (b == B - 1) *d_count = min(o + counts[b], capacity);
  }
  __syncthreads();
  const int n = s_off + tid;
  if (tid < counts[b] && n < capacity) {
    const int vox = top_idx[b * kMaxP + tid];
    batch_ids[n] = b;
    czyx[(size_t)n * 3 + 0] = vox / (kS * kS);
    czyx[(size_t)n * 3 + 1] = (vox / kS) % kS;
    czyx[(size_t)n * 3 + 2] = vox % kS;
    conf[n] = top_val[b * kMaxP + tid];
  }
}

// ---------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) bev_regress_kernel(BevDev m, const float* __restrict__ maps_fv, const void* __restrict__ bv,
                                                          int bv_dtype, const void* __restrict__ fv, int fv_dtype,
                                                          const int* __restrict__ d_count, const long long* __restrict__ batch_ids,
                                                          const long long* __restrict__ czyx, float* __restrict__ params_pred,
                                                          long long* __restrict__ cam_czyx) {
  const int n = blockIdx.x, tid = threadIdx.x;
  if (n >= *d_count) return;
  __shared__ float s_in[3][125];
  __shared__ float s_t1[3][27];
  __shared__ float s_cam[3];
  __shared__ int s_c[3];
  __shared__ float s_f[128], s_h1[512], s_h2[512];
  const int b = (int)batch_ids[n], z = (int)czyx[n * 3], y = (int)czyx[n * 3 + 1], x = (int)czyx[n * 3 + 2];
  // cam_maps_3d input field on the 5^3 neighbourhood: coordmap + cam_offset (+ bird's-eye offset on the last component)
  for (int t = tid; t < 375; t += 256) {
    const int c = t / 125, r = t % 125;
    const int zz = z + r / 25 - 2, yy = y + (r / 5) % 5 - 2, xx = x + r % 5 - 2;
    float v = 0.f;                                                  // zero padding of the 3-D conv
    if (zz >= 0 && zz < kD && yy >= 0 && yy < kS && xx >= 0 && xx < kS) {
      v = m.coordmap[(((size_t)zz * kS + yy) * kS + xx) * 3 + c] + maps_fv[(((size_t)b * 4 + 1 + c) * kS + yy) * kS + xx];
      if (c == 2) v += load_as_float(bv, ((size_t)b * kS + xx) * kS + 64 + zz, bv_dtype);   // bev/model.py:212
    }
    s_in[c][r] = v;
  }
  __syncthreads();
  if (tid < 81) {       // t1 = relu(bn1(conv1)) at the 27 neighbours (zero outside the volume: conv2's padding)
    const int c1 = tid / 27, nb = tid % 27;
    const int nz = nb / 9 - 1, ny = (nb / 3) % 3 - 1, nx = nb % 3 - 1;
    float acc = 0.f;
    if (z + nz >= 0 && z + nz < kD && y + ny >= 0 && y + ny < kS && x + nx >= 0 && x + nx < kS) {
      acc = m.cam_ref[243 + c1];
      for (int c0 = 0; c0 < 3; ++c0)
        for (int tz = 0; tz < 3; ++tz)
          for (int ty = 0; ty < 3; ++ty)
            for (int tx = 0; tx < 3; ++tx)
              acc = fmaf(m.cam_ref[(c1 * 3 + c0) * 27 + tz * 9 + ty * 3 + tx],
                         s_in[c0][(nz + tz + 1) * 25 + (ny + ty + 1) * 5 + (nx + tx + 1)], acc);
      acc = fmaxf(acc, 0.f);
    }
    s_t1[c1][nb] = acc;
  }
  __syncthreads();
  if (tid < 3) {
    float acc = m.cam_ref[489 + tid];
    for (int c1 = 0; c1 < 3; ++c1)
      for (int t = 0; t < 27; ++t) acc = fmaf(m.cam_ref[246 + (tid * 3 + c1) * 27 + t], s_t1[c1][t], acc);
    s_cam[tid] = acc + s_in[tid][62];                                 // residual of BasicBlock_3D, centre voxel
  }
  __syncthreads();
  if (tid == 0) {       // convert_cam_params_to_centermap_coords + denormalize_center, bev/model.py:89-102
    int best = 0;
    float bd = fabsf(s_cam[0] - m.anchors[0]);
    for (int k = 1; k < 64; ++k) {
      const float dd = fabsf(s_cam[0] - m.anchors[k]);
      if (dd < bd) { bd = dd; best = k; }
    }
    const float c0 = (((float)best / 128.f * 2.f - 1.f) + 1.f) / 2.f * 128.f;
    const float c1 = (s_cam[1] + 1.f) / 2.f * 128.f, c2 = (s_cam[2] + 1.f) / 2.f * 128.f;
    s_c[0] = (int)fminf(fmaxf(c0, 1.f), 127.f);
    s_c[1] = (int)fminf(fmaxf(c1, 1.f), 127.f);
    s_c[2] = (int)fminf(fmaxf(c2, 1.f), 127.f);
    cam_czyx[n * 3] = s_c[0]; cam_czyx[n * 3 + 1] = s_c[1]; cam_czyx[n * 3 + 2] = s_c[2];
  }
  __syncthreads();
  if (tid < 128)       // feature[b,:,cy,cx] + position_embeddings(cz), bev/model.py:217-223
    s_f[tid] = load_as_float(fv, (((size_t)b * kS + s_c[1]) * kS + s_c[2]) * 128 + tid, fv_dtype) + m.embed[s_c[0] * 128 + tid];
  __syncthreads();
  for (int j = tid; j < 512; j += 256) {
    float acc = m.b0[j];
    for (int k = 0; k < 128; ++k) acc = fmaf(m.w0t[k * 512 + j], s_f[k], acc);
    s_h1[j] = fmaxf(acc, 0.f);
  }
  __syncthreads();
  for (int j = tid; j < 512; j += 256) {
    float acc = m.b1[j];
    for (int k = 0; k < 512; ++k) acc = fmaf(m.w1t[k * 512 + j], s_h1[k], acc);
    s_h2[j] = fmaxf(acc, 0.f);
  }
  __syncthreads();
  if (tid < 143) {
    float acc = m.b2[tid];
    for (int k = 0; k < 512; ++k) acc = fmaf(m.w2t[k * 143 + tid], s_h2[k], acc);
    params_pred[(size_t)n * 146 + 3 + tid] = acc;
  }
  if (tid < 3) params_pred[(size_t)n * 146 + tid] = s_cam[tid];
}

__global__ void __launch_bounds__(64) bev_unpack_kernel(const float* __restrict__ params_pred, const int* __restrict__ d_count,
                                                        float* __restrict__ cam, float* __restrict__ thetas,
                                                        float* __restrict__ betas, float* __restrict__ cam_trans) {
  const int n = blockIdx.x, tid = threadIdx.x;
  if (n >= *d_count) return;
  __shared__ float s_row[146];
  for (int i = tid; i < 146; i += 64) s_row[i] = params_pred[(size_t)n * 146 + i];
  __syncthreads();
  if (tid < 22) {
    float aa[3];
    rot6d_to_aa(&s_row[3 + tid * 6], aa);
    thetas[(size_t)n * 72 + tid * 3] = aa[0]; thetas[(size_t)n * 72 + tid * 3 + 1] = aa[1]; thetas[(size_t)n * 72 + tid * 3 + 2] = aa[2];
  } else if (tid < 28) {
    thetas[(size_t)n * 72 + 66 + tid - 22] = 0.f;
  } else if (tid < 31) {
    cam[n * 3 + tid - 28] = s_row[tid - 28];
  } else if (tid >= 32 && tid < 43) {
    betas[(size_t)n * 11 + tid - 32] = s_row[135 + tid - 32];
  } else if (tid == 48) {       // denormalize_cam_params_to_trans, bev/post_parser.py:114-128
    const float depth = 1.f / (s_row[0] * kTanFov + 1e-3f);
    cam_trans[n * 3 + 0] = s_row[2] * depth * kTanFov;
    cam_trans[n * 3 + 1] = s_row[1] * depth * kTanFov;
    cam_trans[n * 3 + 2] = depth;
  }
}

__global__ void __launch_bounds__(256) bev_merge_smil_kernel(const float* __restrict__ betas, const int* __restrict__ d_count,
                                                             const float* __restrict__ verts_smil, const float* __restrict__ joints_smil,
                                                             float* __restrict__ verts, float* __restrict__ joints) {
  const int n = blockIdx.x;
  if (n >= *d_count || !(betas[(size_t)n * 11 + 10] > 0.8f)) return;      // baby_thresh, bev/post_parser.py:260,263
  for (int i = blockIdx.y * 256 + threadIdx.x; i < 6890 * 3; i += gridDim.y * 256) verts[(size_t)n * 20670 + i] = verts_smil[(size_t)n * 20670 + i];
  if (blockIdx.y == 0)
    for (int i = threadIdx.x; i < 213; i += 256) joints[(size_t)n * 213 + i] = joints_smil[(size_t)n * 213 + i];
}

// pad_tab (device [B,6] fp32 [top,bottom,left,right,h,w] per frame, may be NULL): person n projects with the row of its
// frame batch_ids[n] instead of the shared size / left / top
__global__ void __launch_bounds__(128) bev_project_kernel(const float* __restrict__ joints, const float* __restrict__ cam_trans,
                                                          const int* __restrict__ d_count, float size, float left, float top,
                                                          const float* __restrict__ pad_tab, const long long* __restrict__ batch_ids,
                                                          float* __restrict__ pj2d_org) {
  const int n = blockIdx.x, j = threadIdx.x;
  if (n >= *d_count || j >= 71) return;
  if (pad_tab) {
    const float* f = pad_tab + batch_ids[n] * 6;
    top = f[0]; left = f[2];
    size = f[4] > f[5] ? f[4] : f[5];
  }
  const float* q = joints + ((size_t)n * 71 + j) * 3;
  const float px = q[0] + cam_trans[n * 3], py = q[1] + cam_trans[n * 3 + 1], pz = q[2] + cam_trans[n * 3 + 2];
  const float iz = pz + 1e-6f;
  const float u = (px / iz) * 443.4f / 256.f, v = (py / iz) * 443.4f / 256.f;     // bev/post_parser.py:95-105
  pj2d_org[((size_t)n * 71 + j) * 2 + 0] = (u + 1.f) * size / 2.f - left;          // :132-133
  pj2d_org[((size_t)n * 71 + j) * 2 + 1] = (v + 1.f) * size / 2.f - top;
}

// [start, start + n) = the rows of frame b (rows are grouped by frame, in frame order); n capped at cap
__device__ __forceinline__ void frame_rows(const long long* __restrict__ batch_ids, int N, int b, int* s_start, int* s_n, int cap = kMaxP) {
  int s = 0;
  while (s < N && batch_ids[s] < b) ++s;
  int e = s;
  while (e < N && batch_ids[e] == b) ++e;
  *s_start = s; *s_n = min(e - s, cap);
}

// Both reference post-filters on one frame's (<= CAP) persons [st, st + nf), by the whole CTA (256 threads).  Persons with
// s_drop[i] set on entry take part in neither filter (the long-image boundary drop).  On return s_removed[i] = 1 for every
// person that is dropped or filtered out.
//   suppressing_redundant_prediction_via_projection (bev/post_parser.py:167-198): every pair below the threshold at once;
//     conf == nullptr removes the smaller scale (cam[:,0]) of the pair, else the lower center_confs (conf_based=True, :191-193);
//     on a tie the later person
//   remove_outlier(relative_scale_thresh, scale_thresh) (:200-222)
template <int CAP = kMaxP>
__device__ void postfilter_frame(const float* __restrict__ pj2d_org, const float* __restrict__ cam, const float* __restrict__ cam_trans,
                                 const float* __restrict__ conf, int st, int nf, float nms_thr_px, float rel_scale_thresh,
                                 float scale_thresh, const int* s_drop, int* s_removed, int* s_kept, float* s_mean, int* s_nk) {
  const int tid = threadIdx.x;
  if (tid < CAP) s_removed[tid] = tid < nf ? s_drop[tid] : 0;
  __syncthreads();
  if (nf > 1) {
    for (int pr = tid; pr < nf * nf; pr += blockDim.x) {
      const int i = pr / nf, j = pr % nf;
      if (i >= j || s_drop[i] || s_drop[j]) continue;
      const float* a = pj2d_org + (size_t)(st + i) * 142;
      const float* c = pj2d_org + (size_t)(st + j) * 142;
      float sum = 0.f;
      for (int k = 0; k < 71; ++k) {
        const float dx = a[2 * k] - c[2 * k], dy = a[2 * k + 1] - c[2 * k + 1];
        sum += sqrtf(dx * dx + dy * dy);
      }
      const float si = cam[(st + i) * 3] * 2.f, sj = cam[(st + j) * 3] * 2.f;
      if (sum / 71.f / fmaxf(si, sj) < nms_thr_px) {
        const bool first = conf ? conf[st + i] < conf[st + j] : si < sj;
        atomicExch(&s_removed[first ? i : j], 1);
      }
    }
  }
  __syncthreads();
  if (tid == 0) {
    int k = 0;
    for (int i = 0; i < nf; ++i)
      if (!s_removed[i]) s_kept[k++] = i;
    *s_nk = k;
  }
  __syncthreads();
  const int nk = *s_nk;
  if (nk >= 3) {
    if (tid < nk) {
      const float* ti = cam_trans + (size_t)(st + s_kept[tid]) * 3;
      float sum = 0.f, mn = CUDART_INF_F, mx = -CUDART_INF_F;
      for (int j = 0; j < nk; ++j) {
        const float* tj = cam_trans + (size_t)(st + s_kept[j]) * 3;
        const float dx = ti[0] - tj[0], dy = ti[1] - tj[1], dz = ti[2] - tj[2];
        const float d = sqrtf(dx * dx + dy * dy + dz * dz);
        sum += d; mn = fminf(mn, d); mx = fmaxf(mx, d);
      }
      s_mean[tid] = (sum - mn - mx) / (float)(nk - 2);       // sorted row without its first and last entry
    }
    __syncthreads();
    if (tid < nk) {
      float tot = 0.f;
      for (int j = 0; j < nk; ++j) tot += s_mean[j];
      const float rel = s_mean[tid] / ((tot - s_mean[tid]) / (float)(nk - 1));
      if (rel > rel_scale_thresh && cam[(st + s_kept[tid]) * 3] < scale_thresh) s_removed[s_kept[tid]] = 1;
    }
    __syncthreads();
  }
}

// one CTA per frame: both reference post-filters on that frame's (<= CAP) persons, then flags for the survivors.  CAP is
// 64 for the regressor's rows and 128 for the rows of BEV's video mode (two rows per detection at most)
template <int CAP>
__global__ void __launch_bounds__(256) bev_postfilter_kernel(const float* __restrict__ pj2d_org, const float* __restrict__ cam,
                                                             const float* __restrict__ cam_trans, const long long* __restrict__ batch_ids,
                                                             const int* __restrict__ d_count, float nms_thr_px, float rel_scale_thresh,
                                                             const float* __restrict__ pad_tab, float nms_thresh, int* __restrict__ keep) {
  __shared__ int s_start, s_n;
  __shared__ int s_drop[CAP], s_removed[CAP], s_kept[CAP], s_nk;
  __shared__ float s_mean[CAP];
  const int b = blockIdx.x, tid = threadIdx.x;
  if (pad_tab) {                       // this frame's own threshold nms_thresh * max(h, w) / 640 (bev/post_parser.py:186-187)
    const float h = pad_tab[b * 6 + 4], w = pad_tab[b * 6 + 5];
    nms_thr_px = __fdiv_rn(__fmul_rn(nms_thresh, h > w ? h : w), 640.f);
  }
  if (tid == 0) frame_rows(batch_ids, *d_count, b, &s_start, &s_n, CAP);
  if (tid < CAP) s_drop[tid] = 0;
  __syncthreads();
  const int st = s_start, nf = s_n;
  if (nf == 0) return;
  postfilter_frame<CAP>(pj2d_org, cam, cam_trans, nullptr, st, nf, nms_thr_px, rel_scale_thresh, 0.25f, s_drop, s_removed, s_kept, s_mean, &s_nk);
  if (tid < nf) keep[st + tid] = s_removed[tid] ? 0 : 1;
}

// ---------------------------------------------------------------------------------------------------------
// Long-image (crowd) mode, bev/main.py:184-258.  Per-crop table row (fp32, one per crop of the image):
//   [0] drop persons with cam x > this (1 - ratio(i), +inf for the last crop)             main.py:209-215, split2process.py:41-46
//   [1] drop persons with cam x < this (ratio(i-1) - 1 for crops 2.., -inf for crops 0, 1)  :221-226
//   [2] projection size max(ch, cw) (offsets [0, ch, 0, cw, ch, cw])                        :216-217
//   [3] suppression threshold in pixels, nms_thresh * max(ch, cw) / 640                      :231
//   [4] cam scale max(r-l, b-t) / max(h, w), [5] cam x shift mean(l, r) / (w/2) - 1          split2process.py:48-58
constexpr int kCropTab = 6;

// one CTA per crop of the chunk: boundary drop, projection to crop pixels, conf-based suppression, remove_outlier with
// scale_thresh 1, then keep flags and the full-image cam of every person
__global__ void __launch_bounds__(256) bev_crop_filter_kernel(const float* __restrict__ joints, const float* __restrict__ cam,
                                                              const float* __restrict__ cam_trans, const float* __restrict__ conf,
                                                              const long long* __restrict__ batch_ids, const int* __restrict__ d_count,
                                                              const float* __restrict__ crop_table, int crop0, float rel_scale_thresh,
                                                              float* __restrict__ pj2d, int* __restrict__ keep,
                                                              float* __restrict__ cam_full) {
  __shared__ int s_start, s_n;
  __shared__ int s_drop[kMaxP], s_removed[kMaxP], s_kept[kMaxP], s_nk;
  __shared__ float s_mean[kMaxP];
  const int b = blockIdx.x, tid = threadIdx.x;
  if (tid == 0) frame_rows(batch_ids, *d_count, b, &s_start, &s_n);
  __syncthreads();
  const int st = s_start, nf = s_n;
  if (nf == 0) return;
  const float* tab = crop_table + (size_t)(crop0 + b) * kCropTab;
  if (tid < nf) {
    const float x = cam[(st + tid) * 3 + 2];
    s_drop[tid] = (x > tab[0] || x < tab[1]) ? 1 : 0;
  }
  const float size = tab[2];
  for (int t = tid; t < nf * 71; t += 256) {       // perspective_projection + convert_proejection_from_input_to_orgimg
    const int n = st + t / 71, j = t % 71;
    const float* q = joints + ((size_t)n * 71 + j) * 3;
    const float px = q[0] + cam_trans[n * 3], py = q[1] + cam_trans[n * 3 + 1], pz = q[2] + cam_trans[n * 3 + 2];
    const float iz = pz + 1e-6f;
    const float u = (px / iz) * 443.4f / 256.f, v = (py / iz) * 443.4f / 256.f;
    pj2d[((size_t)n * 71 + j) * 2 + 0] = (u + 1.f) * size / 2.f;
    pj2d[((size_t)n * 71 + j) * 2 + 1] = (v + 1.f) * size / 2.f;
  }
  __syncthreads();
  postfilter_frame(pj2d, cam, cam_trans, conf, st, nf, tab[3], rel_scale_thresh, 1.f, s_drop, s_removed, s_kept, s_mean, &s_nk);
  if (tid < nf) {
    const int n = st + tid;
    keep[n] = s_removed[tid] ? 0 : 1;
    // convert_crop_cam_params2full_image: cam *= scale (all three), then cam[:,2] += shift, fp32 like the in-place torch ops
    const float s = tab[4];
    cam_full[n * 3 + 0] = __fmul_rn(cam[n * 3 + 0], s);
    cam_full[n * 3 + 1] = __fmul_rn(cam[n * 3 + 1], s);
    cam_full[n * 3 + 2] = __fadd_rn(__fmul_rn(cam[n * 3 + 2], s), tab[5]);
  }
}

// Stable compaction by one CTA (blockDim a multiple of 32, <= 1024): out[k] = val(i) for the k-th i < n with flag(i); returns
// the count to every thread.
template <class Flag, class Val>
__device__ int block_compact(int n, Flag flag, Val val, int* __restrict__ out) {
  __shared__ int s_warp[32], s_base, s_tot;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5, nw = blockDim.x >> 5;
  if (tid == 0) s_base = 0;
  __syncthreads();
  for (int c = 0; c < n; c += blockDim.x) {
    const int i = c + tid;
    const bool f = i < n && flag(i);
    const unsigned m = __ballot_sync(0xffffffffu, f);
    if (lane == 0) s_warp[wid] = __popc(m);
    __syncthreads();
    if (wid == 0) {
      const int v = lane < nw ? s_warp[lane] : 0;
      int inc = v;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int u = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += u;
      }
      if (lane < nw) s_warp[lane] = inc - v;
      if (lane == 31) s_tot = inc;
    }
    __syncthreads();
    if (f) out[s_base + s_warp[wid] + __popc(m & ((1u << lane) - 1u))] = val(i);
    __syncthreads();
    if (tid == 0) s_base += s_tot;
    __syncthreads();
  }
  return s_base;
}

// append the chunk's survivors at the image's running count acc_count[0]: sel = their chunk rows, ctl = {base, n_new}
__global__ void __launch_bounds__(1024) bev_crop_append_kernel(const int* __restrict__ keep, const int* __restrict__ d_count,
                                                               int acc_capacity, int* __restrict__ acc_count, int* __restrict__ sel,
                                                               int* __restrict__ ctl) {
  const int N = *d_count;
  const int k = block_compact(N, [&](int i) { return keep[i] != 0; }, [](int i) { return i; }, sel);
  if (threadIdx.x == 0) {
    const int base = *acc_count, n = min(k, acc_capacity - base);
    ctl[0] = base; ctl[1] = n;
    acc_count[0] = base + n;
    acc_count[1] += N;                    // persons detected in the image so far, survivors or not
  }
}

__global__ void __launch_bounds__(256) append_rows_kernel(const uint32_t* __restrict__ src, int row_words, const int* __restrict__ sel,
                                                          const int* __restrict__ ctl, uint32_t* __restrict__ dst) {
  const int i = blockIdx.x;
  if (i >= ctl[1]) return;
  const uint32_t* s = src + (size_t)sel[i] * row_words;
  uint32_t* d = dst + (size_t)(ctl[0] + i) * row_words;
  for (int k = blockIdx.y * 256 + threadIdx.x; k < row_words; k += gridDim.y * 256) d[k] = s[k];
}

// merged stage, bev/main.py:253-256: cam_trans from the full-image cam and projection with the full image's pad info
__global__ void __launch_bounds__(128) bev_long_project_kernel(const float* __restrict__ cam, const float* __restrict__ joints,
                                                               const int* __restrict__ d_count, float size, float left, float top,
                                                               float* __restrict__ cam_trans, float* __restrict__ pj2d_org,
                                                               int* __restrict__ removed) {
  const int n = blockIdx.x, j = threadIdx.x;
  if (n >= *d_count) return;
  float tr[3];
  bev_cam_trans_rn(cam + n * 3, tr);                    // denormalize_cam_params_to_trans (bev/post_parser.py:114-128)
  const float tx = tr[0], ty = tr[1], depth = tr[2];
  if (j == 0) {
    cam_trans[n * 3 + 0] = tx; cam_trans[n * 3 + 1] = ty; cam_trans[n * 3 + 2] = depth;
    removed[n] = 0;
  }
  if (j >= 71) return;
  const float* q = joints + ((size_t)n * 71 + j) * 3;
  const float iz = q[2] + depth + 1e-6f;
  const float u = ((q[0] + tx) / iz) * 443.4f / 256.f, v = ((q[1] + ty) / iz) * 443.4f / 256.f;
  pj2d_org[((size_t)n * 71 + j) * 2 + 0] = (u + 1.f) * size / 2.f - left;
  pj2d_org[((size_t)n * 71 + j) * 2 + 1] = (v + 1.f) * size / 2.f - top;
}

// conf-based suppression over ALL accumulated persons (not bounded by 64): one 16 x 16 tile of pairs (i < j) per CTA; every
// pair below the threshold removes its lower-confidence member, all pairs at once like the reference's torch.where
constexpr int kPT = 16;
__global__ void __launch_bounds__(256) bev_long_pairs_kernel(const float* __restrict__ pj2d_org, const float* __restrict__ cam,
                                                             const float* __restrict__ conf, const int* __restrict__ d_count,
                                                             float nms_thr_px, int* __restrict__ removed) {
  __shared__ float s_a[kPT][142], s_b[kPT][142];
  const int N = *d_count;
  const int i0 = blockIdx.y * kPT, j0 = blockIdx.x * kPT;
  if (i0 >= N || j0 >= N || j0 + kPT - 1 <= i0) return;
  for (int t = threadIdx.x; t < kPT * 142; t += 256) {
    const int r = t / 142, c = t % 142;
    s_a[r][c] = i0 + r < N ? pj2d_org[(size_t)(i0 + r) * 142 + c] : 0.f;
    s_b[r][c] = j0 + r < N ? pj2d_org[(size_t)(j0 + r) * 142 + c] : 0.f;
  }
  __syncthreads();
  const int ii = threadIdx.x / kPT, jj = threadIdx.x % kPT, i = i0 + ii, j = j0 + jj;
  if (i >= N || j >= N || i >= j) return;
  float sum = 0.f;
  for (int k = 0; k < 71; ++k) {
    const float dx = s_a[ii][2 * k] - s_b[jj][2 * k], dy = s_a[ii][2 * k + 1] - s_b[jj][2 * k + 1];
    sum += sqrtf(dx * dx + dy * dy);
  }
  const float si = cam[i * 3] * 2.f, sj = cam[j * 3] * 2.f;
  if (sum / 71.f / fmaxf(si, sj) < nms_thr_px) removed[conf[i] < conf[j] ? i : j] = 1;
}

// survivors of the suppression: ws_sel[0, nk), *ws_nk = nk
__global__ void __launch_bounds__(1024) bev_long_kept_kernel(const int* __restrict__ removed, const int* __restrict__ d_count,
                                                             int* __restrict__ ws_sel, int* __restrict__ ws_nk) {
  const int k = block_compact(*d_count, [&](int i) { return removed[i] == 0; }, [](int i) { return i; }, ws_sel);
  if (threadIdx.x == 0) *ws_nk = k;
}

// remove_outlier, mean of each survivor's sorted distance row without its first and last entry: one CTA per survivor
__global__ void __launch_bounds__(128) bev_long_meandist_kernel(const float* __restrict__ cam_trans, const int* __restrict__ ws_sel,
                                                                const int* __restrict__ ws_nk, float* __restrict__ ws_mean) {
  const int nk = *ws_nk, r = blockIdx.x;
  if (nk < 3 || r >= nk) return;
  const float* ti = cam_trans + (size_t)ws_sel[r] * 3;
  float sum = 0.f, mn = CUDART_INF_F, mx = -CUDART_INF_F;
  for (int k = threadIdx.x; k < nk; k += 128) {
    const float* tj = cam_trans + (size_t)ws_sel[k] * 3;
    const float dx = ti[0] - tj[0], dy = ti[1] - tj[1], dz = ti[2] - tj[2];
    const float d = sqrtf(dx * dx + dy * dy + dz * dz);
    sum += d; mn = fminf(mn, d); mx = fmaxf(mx, d);
  }
  __shared__ float s_sum[4], s_mn[4], s_mx[4];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    sum += __shfl_xor_sync(0xffffffffu, sum, o);
    mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, o));
    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  }
  if ((threadIdx.x & 31) == 0) { s_sum[threadIdx.x >> 5] = sum; s_mn[threadIdx.x >> 5] = mn; s_mx[threadIdx.x >> 5] = mx; }
  __syncthreads();
  if (threadIdx.x == 0) {
    const float s = s_sum[0] + s_sum[1] + s_sum[2] + s_sum[3];
    const float lo = fminf(fminf(s_mn[0], s_mn[1]), fminf(s_mn[2], s_mn[3])), hi = fmaxf(fmaxf(s_mx[0], s_mx[1]), fmaxf(s_mx[2], s_mx[3]));
    ws_mean[r] = (s - lo - hi) / (float)(nk - 2);
  }
}

// relative scale of every survivor against the others, outliers (and cam[:,0] < scale_thresh) removed, final compaction
__global__ void __launch_bounds__(1024) bev_long_outlier_kernel(const float* __restrict__ cam, const int* __restrict__ ws_sel,
                                                                const int* __restrict__ ws_nk, const float* __restrict__ ws_mean,
                                                                float rel_scale_thresh, float scale_thresh, int* __restrict__ sel,
                                                                int* __restrict__ d_count_out) {
  __shared__ float s_part[32];
  __shared__ float s_tot;
  const int nk = *ws_nk, tid = threadIdx.x;
  float tot = 0.f;
  if (nk >= 3) {
    for (int k = tid; k < nk; k += blockDim.x) tot += ws_mean[k];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) tot += __shfl_xor_sync(0xffffffffu, tot, o);
    if ((tid & 31) == 0) s_part[tid >> 5] = tot;
    __syncthreads();
    if (tid == 0) {
      float t = 0.f;
      for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t += s_part[w];
      s_tot = t;
    }
    __syncthreads();
    tot = s_tot;
  }
  auto keep = [&](int k) {
    if (nk < 3) return true;
    const float rel = ws_mean[k] / ((tot - ws_mean[k]) / (float)(nk - 1));
    return !(rel > rel_scale_thresh && cam[ws_sel[k] * 3] < scale_thresh);
  };
  const int n = block_compact(nk, keep, [&](int k) { return ws_sel[k]; }, sel);
  if (tid == 0) *d_count_out = n;
}

__global__ void bev_compact_kernel(const int* __restrict__ keep, const int* __restrict__ d_count, int* __restrict__ sel,
                                   int* __restrict__ d_count_out) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  const int N = *d_count;
  int k = 0;
  for (int i = 0; i < N; ++i)
    if (keep[i]) sel[k++] = i;
  *d_count_out = k;
}

__global__ void __launch_bounds__(256) gather_rows_kernel(const uint32_t* __restrict__ src, int row_words, const int* __restrict__ sel,
                                                          const int* __restrict__ d_count, uint32_t* __restrict__ dst) {
  const int i = blockIdx.x;
  if (i >= *d_count) return;
  const uint32_t* s = src + (size_t)sel[i] * row_words;
  uint32_t* d = dst + (size_t)i * row_words;
  for (int k = blockIdx.y * 256 + threadIdx.x; k < row_words; k += gridDim.y * 256) d[k] = s[k];
}

}  // namespace b200romp

using namespace b200romp;

struct b200romp_bev {
  int device = 0;
  BevDev dev;
  std::vector<void*> allocs;
};

static const float* up(b200romp_bev* h, const float* host, size_t n, bool* ok) {
  void* d = nullptr;
  if (cudaMalloc(&d, n * sizeof(float)) != cudaSuccess || cudaMemcpy(d, host, n * sizeof(float), cudaMemcpyHostToDevice) != cudaSuccess) {
    *ok = false;
    return nullptr;
  }
  h->allocs.push_back(d);
  return reinterpret_cast<const float*>(d);
}

extern "C" {

b200romp_bev* b200romp_bev_create(int device, const b200romp_bev_weights* w) {
  if (!w || !w->center_ref || !w->cam_ref || !w->coordmap || !w->anchors || !w->embed || !w->w0 || !w->b0 || !w->w1 || !w->b1 ||
      !w->w2 || !w->b2) {
    set_error("bev_create: null weight pointer");
    return nullptr;
  }
  if (cudaSetDevice(device) != cudaSuccess) {
    set_error("bev_create: cudaSetDevice(%d) failed (no CPU fallback)", device);
    return nullptr;
  }
  b200romp_bev* h = new b200romp_bev();
  h->device = device;
  bool ok = true;
  auto transpose = [](const float* src, int rows, int cols) {      // [rows][cols] -> [cols][rows]
    std::vector<float> t((size_t)rows * cols);
    for (int r = 0; r < rows; ++r)
      for (int c = 0; c < cols; ++c) t[(size_t)c * rows + r] = src[(size_t)r * cols + c];
    return t;
  };
  BevDev& d = h->dev;
  d.center_ref = up(h, w->center_ref, 56, &ok);
  d.cam_ref = up(h, w->cam_ref, 492, &ok);
  d.coordmap = up(h, w->coordmap, (size_t)kVol * 3, &ok);
  d.anchors = up(h, w->anchors, 64, &ok);
  d.embed = up(h, w->embed, 128 * 128, &ok);
  std::vector<float> t0 = transpose(w->w0, 512, 128), t1 = transpose(w->w1, 512, 512), t2 = transpose(w->w2, 143, 512);
  d.w0t = up(h, t0.data(), t0.size(), &ok); d.b0 = up(h, w->b0, 512, &ok);
  d.w1t = up(h, t1.data(), t1.size(), &ok); d.b1 = up(h, w->b1, 512, &ok);
  d.w2t = up(h, t2.data(), t2.size(), &ok); d.b2 = up(h, w->b2, 143, &ok);
  if (!ok) {
    set_error("bev_create: upload failed (%s)", cudaGetErrorString(cudaGetLastError()));
    b200romp_bev_destroy(h);
    return nullptr;
  }
  return h;
}

void b200romp_bev_destroy(b200romp_bev* h) {
  if (!h) return;
  cudaSetDevice(h->device);
  for (void* p : h->allocs) cudaFree(p);
  delete h;
}

int b200romp_bev_bv_input(const float* maps_fv, const void* img_feats, int feats_dtype, int feats_C, int batch, void* out, int out_dtype,
                          b200romp_stream stream) {
  B2R_REQUIRE(maps_fv && img_feats && out && batch > 0 && feats_C >= 16, "bev_bv_input: bad arguments");
  const size_t n = (size_t)batch * kS * 2560;
  bev_bv_input_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(maps_fv, img_feats, feats_dtype, feats_C, batch, out, out_dtype);
  B2R_CUDA_OK(cudaGetLastError());
  return B200ROMP_OK;
}

int b200romp_bev_center3d(b200romp_bev* h, const float* maps_fv, const void* bv_out, int bv_dtype, int batch, float* tmp,
                          float* center3d, b200romp_stream stream) {
  B2R_REQUIRE(h && maps_fv && bv_out && tmp && center3d && batch > 0, "bev_center3d: bad arguments");
  B2R_CUDA_OK(cudaSetDevice(h->device));
  static const bool two_pass = [] { const char* e = getenv("B200ROMP_BEV_CENTER3D_2PASS"); return e && e[0] == '1'; }();
  if (two_pass) {                      // round-1 formulation (one thread per voxel, intermediate in `tmp`): kept for A/B checks
    const size_t n = (size_t)batch * kVol;
    const unsigned g = (unsigned)((n + 255) / 256);
    bev_center3d_kernel<<<g, 256, 0, (cudaStream_t)stream>>>(maps_fv, bv_out, bv_dtype, h->dev, batch, nullptr, tmp, 1);
    bev_center3d_kernel<<<g, 256, 0, (cudaStream_t)stream>>>(maps_fv, bv_out, bv_dtype, h->dev, batch, tmp, center3d, 2);
  } else {
    dim3 grid((kS / kTW) * (kS / kTH), kD / kTD, batch);
    bev_center3d_fused_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(maps_fv, bv_out, bv_dtype, h->dev, center3d);
  }
  B2R_CUDA_OK(cudaGetLastError());
  return B200ROMP_OK;
}

long long b200romp_bev_parse_workspace_bytes(int batch) {
  return (long long)batch * (sizeof(int) * 2 + kCandCap * 8 + kMaxP * 8);
}

int b200romp_bev_parse3d(const float* center3d, int batch, float thresh, int capacity, int* d_count, long long* batch_ids,
                         long long* czyx, float* conf, void* workspace, b200romp_stream stream_) {
  B2R_REQUIRE(center3d && d_count && batch_ids && czyx && conf && workspace && batch > 0 && capacity > 0, "bev_parse3d: bad arguments");
  B2R_REQUIRE(thresh >= 0.f, "bev_parse3d: thresh must be >= 0");
  cudaStream_t stream = (cudaStream_t)stream_;
  int* cand_count = reinterpret_cast<int*>(workspace);
  int* counts = cand_count + batch;
  int* cand_idx = counts + batch;
  float* cand_val = reinterpret_cast<float*>(cand_idx + (size_t)batch * kCandCap);
  int* top_idx = reinterpret_cast<int*>(cand_val + (size_t)batch * kCandCap);
  float* top_val = reinterpret_cast<float*>(top_idx + (size_t)batch * kMaxP);
  B2R_CUDA_OK(cudaMemsetAsync(cand_count, 0, sizeof(int) * batch, stream));
  const size_t n = (size_t)batch * kVol;
  bev_nms3d_kernel<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(center3d, batch, thresh, cand_count, cand_idx, cand_val);
  bev_top64_kernel<<<batch, 1024, 0, stream>>>(cand_count, cand_idx, cand_val, counts, top_idx, top_val);
  bev_emit_kernel<<<batch, 64, 0, stream>>>(batch, capacity, counts, top_idx, top_val, d_count, batch_ids, czyx, conf);
  B2R_CUDA_OK(cudaGetLastError());
  return B200ROMP_OK;
}

int b200romp_bev_regress(b200romp_bev* h, const float* maps_fv, const void* bv_out, int bv_dtype, const void* fv_feats, int fv_dtype,
                         int capacity, const int* d_count, const long long* batch_ids, const long long* czyx, float* params_pred,
                         long long* cam_czyx, float* cam, float* thetas, float* betas, float* cam_trans, b200romp_stream stream_) {
  B2R_REQUIRE(h && maps_fv && bv_out && fv_feats && d_count && batch_ids && czyx && params_pred && cam_czyx && cam && thetas &&
                  betas && cam_trans && capacity > 0, "bev_regress: bad arguments");
  B2R_CUDA_OK(cudaSetDevice(h->device));
  cudaStream_t stream = (cudaStream_t)stream_;
  bev_regress_kernel<<<capacity, 256, 0, stream>>>(h->dev, maps_fv, bv_out, bv_dtype, fv_feats, fv_dtype, d_count, batch_ids, czyx,
                                                   params_pred, cam_czyx);
  bev_unpack_kernel<<<capacity, 64, 0, stream>>>(params_pred, d_count, cam, thetas, betas, cam_trans);
  B2R_CUDA_OK(cudaGetLastError());
  return B200ROMP_OK;
}

static int bev_post(const float* betas, const float* verts_smil, const float* joints_smil, float* verts, float* joints, const float* cam,
                    const float* cam_trans, const long long* batch_ids, int batch, int capacity, const int* d_count, const float* offsets6,
                    const float* pad_table, float nms_thresh, float rel_scale_thresh, float img_max_side, float* pj2d_org, int* keep,
                    int* sel, int* d_count_out, cudaStream_t stream) {
  if (verts_smil && joints_smil)
    bev_merge_smil_kernel<<<dim3(capacity, 4), 256, 0, stream>>>(betas, d_count, verts_smil, joints_smil, verts, joints);
  float top = 0.f, left = 0.f, size = 0.f;
  if (offsets6) {
    const float hh = offsets6[4], ww = offsets6[5];
    top = offsets6[0]; left = offsets6[2]; size = hh > ww ? hh : ww;
  }
  bev_project_kernel<<<capacity, 128, 0, stream>>>(joints, cam_trans, d_count, size, left, top, pad_table, batch_ids, pj2d_org);
  B2R_CUDA_OK(cudaMemsetAsync(keep, 0, sizeof(int) * capacity, stream));
  if (capacity > batch * kMaxP)
    bev_postfilter_kernel<2 * kMaxP><<<batch, 256, 0, stream>>>(pj2d_org, cam, cam_trans, batch_ids, d_count,
                                                                nms_thresh * img_max_side / 640.f, rel_scale_thresh, pad_table,
                                                                nms_thresh, keep);
  else
    bev_postfilter_kernel<kMaxP><<<batch, 256, 0, stream>>>(pj2d_org, cam, cam_trans, batch_ids, d_count, nms_thresh * img_max_side / 640.f,
                                                            rel_scale_thresh, pad_table, nms_thresh, keep);
  bev_compact_kernel<<<1, 32, 0, stream>>>(keep, d_count, sel, d_count_out);
  B2R_CUDA_OK(cudaGetLastError());
  return B200ROMP_OK;
}

int b200romp_bev_post(const float* betas, const float* verts_smil, const float* joints_smil, float* verts, float* joints,
                      const float* cam, const float* cam_trans, const long long* batch_ids, int batch, int capacity,
                      const int* d_count, const float* offsets6, float nms_thresh, float rel_scale_thresh, float img_max_side,
                      float* pj2d_org, int* keep, int* sel, int* d_count_out, b200romp_stream stream_) {
  B2R_REQUIRE(betas && verts && joints && cam && cam_trans && batch_ids && d_count && offsets6 && pj2d_org && keep && sel &&
                  d_count_out && batch > 0 && capacity > 0, "bev_post: bad arguments");
  return bev_post(betas, verts_smil, joints_smil, verts, joints, cam, cam_trans, batch_ids, batch, capacity, d_count, offsets6, nullptr,
                  nms_thresh, rel_scale_thresh, img_max_side, pj2d_org, keep, sel, d_count_out, (cudaStream_t)stream_);
}

int b200romp_bev_post_frames(const float* betas, const float* verts_smil, const float* joints_smil, float* verts, float* joints,
                             const float* cam, const float* cam_trans, const long long* batch_ids, int batch, int capacity,
                             const int* d_count, const float* pad_table, float nms_thresh, float rel_scale_thresh, float* pj2d_org,
                             int* keep, int* sel, int* d_count_out, b200romp_stream stream_) {
  B2R_REQUIRE(betas && verts && joints && cam && cam_trans && batch_ids && d_count && pad_table && pj2d_org && keep && sel &&
                  d_count_out && batch > 0 && capacity > 0, "bev_post_frames: bad arguments");
  return bev_post(betas, verts_smil, joints_smil, verts, joints, cam, cam_trans, batch_ids, batch, capacity, d_count, nullptr, pad_table,
                  nms_thresh, rel_scale_thresh, 0.f, pj2d_org, keep, sel, d_count_out, (cudaStream_t)stream_);
}

int b200romp_bev_crop_post(const float* betas, const float* verts_smil, const float* joints_smil, float* verts, float* joints,
                           const float* thetas, const float* params_pred, const float* conf, const float* cam, const float* cam_trans,
                           const long long* batch_ids, int batch, int capacity, const int* d_count, const float* crop_table,
                           int crop0, float rel_scale_thresh, float* pj2d, int* keep, int* sel, float* cam_full, int acc_capacity,
                           int* acc_count, int* acc_ctl, float* acc_verts, float* acc_joints, float* acc_thetas, float* acc_betas,
                           float* acc_params_pred, float* acc_conf, float* acc_cam, b200romp_stream stream_) {
  B2R_REQUIRE(betas && verts && joints && thetas && params_pred && conf && cam && cam_trans && batch_ids && d_count && crop_table &&
                  pj2d && keep && sel && cam_full && acc_count && acc_ctl && acc_verts && acc_joints && acc_thetas && acc_betas &&
                  acc_params_pred && acc_conf && acc_cam && batch > 0 && capacity > 0 && crop0 >= 0 && acc_capacity > 0,
              "bev_crop_post: bad arguments");
  cudaStream_t stream = (cudaStream_t)stream_;
  if (verts_smil && joints_smil)
    bev_merge_smil_kernel<<<dim3(capacity, 4), 256, 0, stream>>>(betas, d_count, verts_smil, joints_smil, verts, joints);
  B2R_CUDA_OK(cudaMemsetAsync(keep, 0, sizeof(int) * capacity, stream));
  bev_crop_filter_kernel<<<batch, 256, 0, stream>>>(joints, cam, cam_trans, conf, batch_ids, d_count, crop_table, crop0,
                                                    rel_scale_thresh, pj2d, keep, cam_full);
  bev_crop_append_kernel<<<1, 1024, 0, stream>>>(keep, d_count, acc_capacity, acc_count, sel, acc_ctl);
  const struct { const void* src; void* dst; int words; } rows[] = {
      {verts, acc_verts, 6890 * 3}, {joints, acc_joints, 71 * 3}, {thetas, acc_thetas, 72}, {betas, acc_betas, 11},
      {params_pred, acc_params_pred, 146}, {conf, acc_conf, 1}, {cam_full, acc_cam, 3}};
  for (const auto& r : rows)
    append_rows_kernel<<<dim3(capacity, r.words > 4096 ? 8 : 1), 256, 0, stream>>>(
        reinterpret_cast<const uint32_t*>(r.src), r.words, sel, acc_ctl, reinterpret_cast<uint32_t*>(r.dst));
  B2R_CUDA_OK(cudaGetLastError());
  return B200ROMP_OK;
}

long long b200romp_bev_long_merge_workspace_bytes(int capacity) { return (long long)capacity * 8 + 16; }

int b200romp_bev_long_merge(const float* cam, const float* joints, const float* conf, int capacity, const int* d_count,
                            const float* offsets6, float nms_thresh, float rel_scale_thresh, float img_max_side, float* cam_trans,
                            float* pj2d_org, int* removed, void* workspace, int* sel, int* d_count_out, b200romp_stream stream_) {
  B2R_REQUIRE(cam && joints && conf && d_count && offsets6 && cam_trans && pj2d_org && removed && workspace && sel && d_count_out &&
                  capacity > 0 && img_max_side > 0.f, "bev_long_merge: bad arguments");
  cudaStream_t stream = (cudaStream_t)stream_;
  int* ws_nk = reinterpret_cast<int*>(workspace);
  int* ws_sel = ws_nk + 4;
  float* ws_mean = reinterpret_cast<float*>(ws_sel + capacity);
  const float top = offsets6[0], left = offsets6[2], hh = offsets6[4], ww = offsets6[5];
  bev_long_project_kernel<<<capacity, 128, 0, stream>>>(cam, joints, d_count, hh > ww ? hh : ww, left, top, cam_trans, pj2d_org, removed);
  const unsigned tiles = (unsigned)((capacity + kPT - 1) / kPT);
  bev_long_pairs_kernel<<<dim3(tiles, tiles), 256, 0, stream>>>(pj2d_org, cam, conf, d_count,
                                                                (float)((double)nms_thresh * img_max_side / 640.0), removed);
  bev_long_kept_kernel<<<1, 1024, 0, stream>>>(removed, d_count, ws_sel, ws_nk);
  bev_long_meandist_kernel<<<capacity, 128, 0, stream>>>(cam_trans, ws_sel, ws_nk, ws_mean);
  bev_long_outlier_kernel<<<1, 1024, 0, stream>>>(cam, ws_sel, ws_nk, ws_mean, rel_scale_thresh, 0.5f, sel, d_count_out);
  B2R_CUDA_OK(cudaGetLastError());
  return B200ROMP_OK;
}

int b200romp_gather_rows(const void* src, int row_bytes, const int* sel, const int* d_count, int capacity, void* dst,
                         b200romp_stream stream) {
  B2R_REQUIRE(src && sel && d_count && dst && row_bytes > 0 && row_bytes % 4 == 0 && capacity > 0, "gather_rows: bad arguments");
  const int words = row_bytes / 4;
  gather_rows_kernel<<<dim3(capacity, words > 4096 ? 8 : 1), 256, 0, (cudaStream_t)stream>>>(
      reinterpret_cast<const uint32_t*>(src), words, sel, d_count, reinterpret_cast<uint32_t*>(dst));
  B2R_CUDA_OK(cudaGetLastError());
  return B200ROMP_OK;
}

}  // extern "C"
