// BEV's video mode (simple_romp/bev/main.py:109-121,165-169,260-287, --temporal_optimize): the reference's 3-D-centre
// ByteTrack (simple_romp/tracker/byte_tracker_3dcenter.py "BT", kalman_filter_3dcenter.py "KF", matching.py), the
// per-(signal, track) One-Euro filters and cam_trans from the smoothed cam, as one kernel per batch placed between
// the BEV regressor and SMPL-A.  One CTA steps the instance's tracker through the batch's frames in batch order;
// threads parallelise over tracks, detections, row channels.  Tracker state is fp64 and stays in device memory.
// Stream mode (a streams handle): one tracker per stream, one CTA per stream present in the batch, each walking its
// stream's frames with the same per-frame step (bev_track_walk); the rows land in per-frame windows and one more small
// kernel compacts them in frame order.
//
// Per frame with at least one detection (bev/main.py:159-166; a frame with nobody does not step the tracker):
//   tracking points [(cam2+1)*128, (cam1+1)*128, cam_trans2*30, cam0*128/2] in fp32 (:269-272), scores against 0.12 /
//   0.05 in fp32 (BT:31-33); Kalman predict of the activated tracked + lost tracks (BT:56-58, lost ones with mean[7]=0);
//   the three associations with thresholds 300 / 600 / 900 (BT:59-112; the second one against the HIGH-score
//   detections, BT:75-80); new tracks (activated at once only on frame 1, BT:246-247); removal after 60 lost frames;
//   the list updates incl. sub_stracks against the removed list of earlier frames (BT:129-137); duplicate removal at 60
//   in 2-D (BT:187-201); one output row per activated tracked track with the nearest detection (BT:149-159, two rows
//   may share a detection); gather of the rows; One-Euro smoothing (romp/utils.py:188-270); cam_trans.
//
// Kalman filter: P stays kron(S, I4) with S = [[a, b], [b, c]] (the initial P, Q and R treat the four axes alike), so a
// track keeps 3 scalars and the gain is closed form.  Assignment: lap.lapjv(cost, extend_cost=True, cost_limit=lam)
// is the minimum-cost (not necessarily perfect) matching with edge costs c - lam; solved here by the Hungarian method
// on the zero-padded k x k matrix min(c - lam, 0), keeping pairs with c < lam (oracle/track_oracle.py:lap_margin).
#include "common.cuh"
#include "rot6d.cuh"
#include "one_euro.cuh"
#include "bev_cam.cuh"
#include <math_constants.h>

namespace b200romp {

constexpr int kTrkMax = 128;              // largest max_tracks
constexpr int kTrkDet = 64;               // detections per frame (BEV's max_person)
constexpr int kTrkThreads = 256;
constexpr int kTracked = 1, kLost = 2, kRemoved = 3;    // basetrack.TrackState (New = 0)
enum { kCtlTracked = 0, kCtlLost, kCtlFrame, kCtlNextId, kCtlBroken, kCtlN };
enum { kMetaId = 0, kMetaState, kMetaAct, kMetaInRemoved, kMetaFrame, kMetaStart, kMetaUsed, kMetaN };

struct TrkDev {
  double* mean;     // [T][8]
  double* S;        // [T][3]  a, b, c of P = kron([[a, b], [b, c]], I4)
  int* meta;        // [T][kMetaN]
  int* lists;       // [2][T]  tracked_stracks, lost_stracks (slots, list order)
  int* ctl;         // [kCtlN]
  float* oe_raw;    // [signals * T][kOeCh]  One-Euro state, slot = signal * T + track slot (show_largest: signal * T)
  float* oe_x;
  float* oe_dx;
  int* oe_seen;     // [signals * T]
  int T, signals;
};

struct TrkSmem {
  double mean[kTrkMax][8];
  double S[kTrkMax][3];
  int meta[kTrkMax][kMetaN];
  int tracked[kTrkMax], lost[kTrkMax], ctl[kCtlN];
  float pts[kTrkDet][4];
  int high[kTrkDet], nh, any_low, st, nf, sig;
  int pool[kTrkMax], npool, unc[kTrkMax], nunc, rows_a[kTrkMax], na, cols[kTrkDet], nc;
  int row_match[kTrkMax], col_match[kTrkDet], rem[kTrkDet], nrem;
  int upd[kTrkMax];                 // detection (frame-local) to update the track with, or -1
  int act[2 * kTrkMax], nact, refind[kTrkMax], nref, lost_new[kTrkMax], nlost_new, rem_new[2 * kTrkMax], nrem_new;
  int new_tracked[3 * kTrkMax], nnt, new_lost[2 * kTrkMax], nnl, dupa[3 * kTrkMax], dupb[2 * kTrkMax];
  int out_slot[2 * kTrkDet], out_det[2 * kTrkDet], nout, out0;
  float R[2 * kTrkDet][9];
  // Hungarian (warp 0)
  double hu[kTrkMax + 1], hv[kTrkMax + 1], hminv[kTrkMax + 1];
  int hp[kTrkMax + 1], hway[kTrkMax + 1], hused[kTrkMax + 1];
};

__device__ __forceinline__ double trk_dist(const double* m, const float* p, int dim) {
  double s = 0.0;
  for (int k = 0; k < dim; ++k) {
    const double d = m[k] - (double)p[k];
    s += d * d;
  }
  return sqrt(s);
}

// Minimum-cost matching of rows_a[0..na) x cols[0..nc) under cost_limit lam: row_match[i] = column index or -1,
// col_match[j] = row index or -1.  cost: [na][nc] in dynamic shared memory.  Called by every thread of the CTA.
__device__ void trk_assign(TrkSmem& s, double* cost, double lam) {
  const int tid = threadIdx.x, n = s.na, m = s.nc;
  for (int e = tid; e < n * m; e += blockDim.x) {
    const int i = e / m, j = e % m;
    cost[e] = trk_dist(s.mean[s.rows_a[i]], s.pts[s.cols[j]], 4);
  }
  for (int i = tid; i < n; i += blockDim.x) s.row_match[i] = -1;
  for (int j = tid; j < m; j += blockDim.x) s.col_match[j] = -1;
  __syncthreads();
  if (n > 0 && m > 0 && tid < 32) {
    const int lane = tid, k = n > m ? n : m;
    auto A = [&](int i, int j) -> double {       // 1-based
      return (i <= n && j <= m) ? fmin(cost[(i - 1) * m + (j - 1)] - lam, 0.0) : 0.0;
    };
    for (int j = lane; j <= k; j += 32) { s.hu[j] = 0.0; s.hv[j] = 0.0; s.hp[j] = 0; s.hway[j] = 0; }
    __syncwarp();
    for (int i = 1; i <= k; ++i) {
      for (int j = lane; j <= k; j += 32) { s.hminv[j] = CUDART_INF; s.hused[j] = 0; }
      if (lane == 0) s.hp[0] = i;
      __syncwarp();
      int j0 = 0;
      do {
        if (lane == 0) s.hused[j0] = 1;
        __syncwarp();
        const int i0 = s.hp[j0];
        double delta = CUDART_INF;
        int j1 = 0x7fffffff;
        for (int j = 1 + lane; j <= k; j += 32) {
          if (s.hused[j]) continue;
          const double cur = A(i0, j) - s.hu[i0] - s.hv[j];
          if (cur < s.hminv[j]) { s.hminv[j] = cur; s.hway[j] = j0; }
          if (s.hminv[j] < delta) { delta = s.hminv[j]; j1 = j; }
        }
        for (int off = 16; off; off >>= 1) {        // argmin, the smallest column on ties (the sequential scan's choice)
          const double od = __shfl_xor_sync(0xffffffffu, delta, off);
          const int oj = __shfl_xor_sync(0xffffffffu, j1, off);
          if (od < delta || (od == delta && oj < j1)) { delta = od; j1 = oj; }
        }
        __syncwarp();
        for (int j = lane; j <= k; j += 32) {
          if (s.hused[j]) { s.hu[s.hp[j]] += delta; s.hv[j] -= delta; }
          else s.hminv[j] -= delta;
        }
        __syncwarp();
        j0 = j1;
      } while (s.hp[j0] != 0);
      if (lane == 0) {
        do { const int j1 = s.hway[j0]; s.hp[j0] = s.hp[j1]; j0 = j1; } while (j0);
      }
      __syncwarp();
    }
    for (int j = 1 + lane; j <= m; j += 32) {
      const int i = s.hp[j] - 1;
      if (i < n && cost[i * m + (j - 1)] - lam < 0.0) { s.row_match[i] = j - 1; s.col_match[j - 1] = i; }
    }
  }
  __syncthreads();
}

// KF.update (:194-224) of track slot t with the measurement p, closed form
__device__ __forceinline__ void trk_kf_update(TrkSmem& s, int t, const float* p) {
  double* m = s.mean[t];
  const double r = 0.05 * m[3], a = s.S[t][0], b = s.S[t][1], c = s.S[t][2];
  const double sa = a + r * r, ka = a / sa, kb = b / sa;
  for (int k = 0; k < 4; ++k) {
    const double in = (double)p[k] - m[k];
    m[k] += ka * in;
    m[4 + k] += kb * in;
  }
  s.S[t][0] = a - ka * ka * sa;
  s.S[t][1] = b - ka * kb * sa;
  s.S[t][2] = c - kb * kb * sa;
}

__device__ __forceinline__ void trk_run_updates(TrkSmem& s) {
  __syncthreads();
  for (int t = threadIdx.x; t < kTrkMax; t += blockDim.x)
    if (s.upd[t] >= 0) { trk_kf_update(s, t, s.pts[s.upd[t]]); s.upd[t] = -1; }
  __syncthreads();
}

struct TrkIn {
  const int* d_count; const long long* batch_ids; const float *conf, *cam, *cam_trans, *thetas, *betas, *params;
  const int* sig_slot; int batch, capacity, show_largest; float smooth_coeff;
};
struct TrkOut {
  int capacity; int* d_count; long long* batch_ids; int *track_ids, *det; float *thetas, *betas, *cam, *cam_trans, *params, *conf;
  int* status;
};

// The walk of one tracker through the batch's frames in order.  stream < 0: the instance's tracker, every frame, filter set
// sig_slot[b], rows appended in frame order, the batch's counts and status written at the end.  stream >= 0 (g offset to
// that stream's state, one filter set): only the frames with sig_slot[b] == stream, frame b's rows written to its window
// [b * 2 * kTrkDet, +nout) for bev_track_compact_kernel; a failed stream marks its frames status[2 + b] = -status.
__device__ void bev_track_walk(TrkSmem& s, double* cost, const TrkDev& g, const TrkIn& in, const TrkOut& out, int stream) {
  const int tid = threadIdx.x, T = g.T;
  for (int i = tid; i < T * 8; i += blockDim.x) s.mean[i / 8][i % 8] = g.mean[i];
  for (int i = tid; i < T * 3; i += blockDim.x) s.S[i / 3][i % 3] = g.S[i];
  for (int i = tid; i < T * kMetaN; i += blockDim.x) s.meta[i / kMetaN][i % kMetaN] = g.meta[i];
  for (int i = tid; i < T; i += blockDim.x) { s.tracked[i] = g.lists[i]; s.lost[i] = g.lists[T + i]; }
  for (int i = tid; i < kTrkMax; i += blockDim.x) s.upd[i] = -1;
  if (tid < kCtlN) s.ctl[tid] = g.ctl[tid];
  if (tid == 0) { s.st = 0; s.out0 = 0; }
  for (int b = tid; b < in.batch; b += blockDim.x)    // rows per frame
    if (stream < 0 || in.sig_slot[b] == stream) out.status[2 + b] = 0;
  __syncthreads();
  const int N = min(*in.d_count, in.capacity);
  int b = 0;
  for (; b < in.batch; ++b) {
    if (s.ctl[kCtlBroken]) break;
    if (stream >= 0 && in.sig_slot[b] != stream) continue;    // another stream's frame
    if (tid == 0) {                                     // rows of frame b (grouped by frame, in frame order)
      int st = s.st;
      while (st < N && in.batch_ids[st] < b) ++st;
      int e = st;
      while (e < N && in.batch_ids[e] == b) ++e;
      s.st = st; s.nf = min(e - st, kTrkDet); s.sig = stream < 0 ? in.sig_slot[b] : 0;
    }
    __syncthreads();
    const int st = s.st, nf = s.nf;
    if (nf == 0) { __syncthreads(); continue; }         // bev/main.py:159-163: no detection, no tracker step
    if (tid < nf) {                                     // bev/main.py:269-272, fp32
      const float* c = in.cam + (size_t)(st + tid) * 3;
      s.pts[tid][0] = __fmul_rn(__fadd_rn(c[2], 1.f), 128.f);
      s.pts[tid][1] = __fmul_rn(__fadd_rn(c[1], 1.f), 128.f);
      s.pts[tid][2] = __fmul_rn(in.cam_trans[(size_t)(st + tid) * 3 + 2], 30.f);
      s.pts[tid][3] = __fmul_rn(c[0], 128.f) / 2.f;
    }
    __syncthreads();
    if (tid == 0) {
      s.nout = 0;
      if (in.show_largest) {                            // bev/main.py:262-267: torch.argmax(cam[:,0]), first on ties
        int best = 0;
        for (int i = 1; i < nf; ++i) if (in.cam[(size_t)(st + i) * 3] > in.cam[(size_t)(st + best) * 3]) best = i;
        s.out_slot[0] = 0; s.out_det[0] = best; s.nout = 1;
      } else {
        ++s.ctl[kCtlFrame];
        s.nh = 0; s.any_low = 0;
        for (int i = 0; i < nf; ++i) {                  // BT:31-37, strict compares in fp32
          const float sc = in.conf[st + i];
          if (sc > 0.12f) s.high[s.nh++] = i;
          if (sc > 0.05f && sc < 0.12f) s.any_low = 1;
        }
        s.nunc = s.npool = 0;                           // BT:47-56
        for (int i = 0; i < s.ctl[kCtlTracked]; ++i) {
          const int t = s.tracked[i];
          if (!s.meta[t][kMetaAct]) s.unc[s.nunc++] = t; else s.pool[s.npool++] = t;
        }
        for (int i = 0; i < s.ctl[kCtlLost]; ++i) s.pool[s.npool++] = s.lost[i];
        s.nact = s.nref = s.nlost_new = s.nrem_new = 0;
        s.na = s.npool;
        for (int i = 0; i < s.npool; ++i) s.rows_a[i] = s.pool[i];
        s.nc = s.nh;
        for (int j = 0; j < s.nh; ++j) s.cols[j] = s.high[j];
      }
    }
    __syncthreads();
    if (!in.show_largest) {
      const int fid = s.ctl[kCtlFrame];
      for (int i = tid; i < s.npool; i += blockDim.x) {  // STrack.multi_predict / KF.multi_predict (:155-192)
        const int t = s.pool[i];
        double* m = s.mean[t];
        if (s.meta[t][kMetaState] != kTracked) m[7] = 0.0;
        const double h = m[3], qp = 0.05 * h, qv = h / 160.0;
        for (int k = 0; k < 4; ++k) m[k] += m[4 + k];
        const double a = s.S[t][0], bb = s.S[t][1], c = s.S[t][2];
        s.S[t][0] = a + 2.0 * bb + c + qp * qp;
        s.S[t][1] = bb + c;
        s.S[t][2] = c + qv * qv;
      }
      __syncthreads();
      trk_assign(s, cost, 300.0);                // first association, BT:59-71
      if (tid == 0) {
        for (int i = 0; i < s.na; ++i) {
          if (s.row_match[i] < 0) continue;
          const int t = s.rows_a[i];
          if (s.meta[t][kMetaState] == kTracked) s.act[s.nact++] = t; else s.refind[s.nref++] = t;
          s.meta[t][kMetaState] = kTracked; s.meta[t][kMetaAct] = 1; s.meta[t][kMetaFrame] = fid;
          s.upd[t] = s.cols[s.row_match[i]];
        }
        int nr = 0;
        s.nrem = 0;                                     // u_detection, for the third association
        for (int j = 0; j < s.nc; ++j) if (s.col_match[j] < 0) s.rem[s.nrem++] = s.cols[j];
        for (int i = 0; i < s.na; ++i)                  // r_tracked_stracks, BT:81
          if (s.row_match[i] < 0 && s.meta[s.rows_a[i]][kMetaState] == kTracked) s.rows_a[nr++] = s.rows_a[i];
        s.na = nr;
        s.nc = s.any_low ? s.nh : 0;                    // BT:75-80: the high-score detections, if any low one exists
        for (int j = 0; j < s.nc; ++j) s.cols[j] = s.high[j];
      }
      trk_run_updates(s);
      trk_assign(s, cost, 600.0);                // second association, BT:81-99
      if (tid == 0) {
        for (int i = 0; i < s.na; ++i) {
          const int t = s.rows_a[i];
          if (s.row_match[i] >= 0) {
            s.act[s.nact++] = t; s.meta[t][kMetaState] = kTracked; s.meta[t][kMetaAct] = 1; s.meta[t][kMetaFrame] = fid;
            s.upd[t] = s.cols[s.row_match[i]];
          } else if (s.meta[t][kMetaState] != kLost) {
            s.meta[t][kMetaState] = kLost; s.lost_new[s.nlost_new++] = t;
          }
        }
        s.na = s.nunc;
        for (int i = 0; i < s.nunc; ++i) s.rows_a[i] = s.unc[i];
        s.nc = s.nrem;
        for (int j = 0; j < s.nrem; ++j) s.cols[j] = s.rem[j];
      }
      trk_run_updates(s);
      trk_assign(s, cost, 900.0);                // unconfirmed tracks, BT:101-112
      if (tid == 0) {
        for (int i = 0; i < s.na; ++i) {
          const int t = s.rows_a[i];
          if (s.row_match[i] >= 0) {
            s.act[s.nact++] = t; s.meta[t][kMetaState] = kTracked; s.meta[t][kMetaAct] = 1; s.meta[t][kMetaFrame] = fid;
            s.upd[t] = s.cols[s.row_match[i]];
          } else {
            s.meta[t][kMetaState] = kRemoved; s.rem_new[s.nrem_new++] = t;
          }
        }
        for (int j = 0; j < s.nc; ++j) {                // new tracks, BT:114-120 / STrack.activate
          if (s.col_match[j] >= 0) continue;
          int t = 0;
          while (t < T && s.meta[t][kMetaUsed]) ++t;
          if (t == T) { s.ctl[kCtlBroken] = 1; break; }
          const float* p = s.pts[s.cols[j]];
          // KF.initiate (:54-86) in the reference's fp32
          const float sp = 0.1f * p[3], sv = 0.0625f * p[3];
          for (int k = 0; k < 4; ++k) { s.mean[t][k] = (double)p[k]; s.mean[t][4 + k] = 0.0; }
          s.S[t][0] = (double)(sp * sp); s.S[t][1] = 0.0; s.S[t][2] = (double)(sv * sv);
          s.meta[t][kMetaId] = ++s.ctl[kCtlNextId];
          s.meta[t][kMetaState] = kTracked; s.meta[t][kMetaAct] = fid == 1; s.meta[t][kMetaInRemoved] = 0;
          s.meta[t][kMetaFrame] = fid; s.meta[t][kMetaStart] = fid; s.meta[t][kMetaUsed] = 1;
          for (int sg = 0; sg < g.signals; ++sg) g.oe_seen[sg * T + t] = 0;     // a new track's filters start fresh
          s.act[s.nact++] = t;
        }
        for (int i = 0; i < s.ctl[kCtlLost]; ++i) {     // BT:122-125
          const int t = s.lost[i];
          if (fid - s.meta[t][kMetaFrame] > 60) { s.meta[t][kMetaState] = kRemoved; s.rem_new[s.nrem_new++] = t; }
        }
        // BT:129-135
        int nt = 0;
        for (int i = 0; i < s.ctl[kCtlTracked]; ++i) if (s.meta[s.tracked[i]][kMetaState] == kTracked) s.new_tracked[nt++] = s.tracked[i];
        auto in_list = [&](int t, int n) { for (int q = 0; q < n; ++q) if (s.new_tracked[q] == t) return true; return false; };
        for (int i = 0; i < s.nact; ++i) if (!in_list(s.act[i], nt)) s.new_tracked[nt++] = s.act[i];
        for (int i = 0; i < s.nref; ++i) if (!in_list(s.refind[i], nt)) s.new_tracked[nt++] = s.refind[i];
        int nl = 0;
        for (int i = 0; i < s.ctl[kCtlLost]; ++i) if (!in_list(s.lost[i], nt)) s.new_lost[nl++] = s.lost[i];
        for (int i = 0; i < s.nlost_new; ++i) s.new_lost[nl++] = s.lost_new[i];
        int nl2 = 0;
        for (int i = 0; i < nl; ++i) if (!s.meta[s.new_lost[i]][kMetaInRemoved]) s.new_lost[nl2++] = s.new_lost[i];
        for (int i = 0; i < s.nrem_new; ++i) s.meta[s.rem_new[i]][kMetaInRemoved] = 1;
        s.nnt = nt; s.nnl = nl2;
      }
      __syncthreads();
      if (s.ctl[kCtlBroken]) break;
      trk_run_updates(s);
      for (int i = tid; i < s.nnt; i += blockDim.x) s.dupa[i] = 0;
      for (int i = tid; i < s.nnl; i += blockDim.x) s.dupb[i] = 0;
      __syncthreads();
      for (int e = tid; e < s.nnt * s.nnl; e += blockDim.x) {   // remove_duplicate_stracks, BT:187-201
        const int p = e / s.nnl, q = e % s.nnl, tp = s.new_tracked[p], tq = s.new_lost[q];
        const double dx = s.mean[tp][0] - s.mean[tq][0], dy = s.mean[tp][1] - s.mean[tq][1];
        if (sqrt(dx * dx + dy * dy) < 60.0) {
          if (s.meta[tp][kMetaFrame] - s.meta[tp][kMetaStart] > s.meta[tq][kMetaFrame] - s.meta[tq][kMetaStart]) s.dupb[q] = 1;
          else s.dupa[p] = 1;
        }
      }
      __syncthreads();
      if (tid == 0) {
        for (int t = 0; t < T; ++t) s.upd[t] = -2;      // -2: not listed any more
        int nt = 0, nl = 0;
        for (int i = 0; i < s.nnt; ++i) if (!s.dupa[i]) { s.tracked[nt++] = s.new_tracked[i]; s.upd[s.new_tracked[i]] = -1; }
        for (int i = 0; i < s.nnl; ++i) if (!s.dupb[i]) { s.lost[nl++] = s.new_lost[i]; s.upd[s.new_lost[i]] = -1; }
        s.ctl[kCtlTracked] = nt; s.ctl[kCtlLost] = nl;
        for (int t = 0; t < T; ++t) { if (s.upd[t] == -2) s.meta[t][kMetaUsed] = 0; s.upd[t] = -1; }
        int no = 0;
        for (int i = 0; i < nt; ++i) if (s.meta[s.tracked[i]][kMetaAct]) s.out_slot[no++] = s.tracked[i];
        s.nout = no;
      }
      __syncthreads();
      for (int r = tid; r < s.nout; r += blockDim.x) {  // get_tracked_ids_byte, BT:149-159: nearest detection, first on ties
        const double* m = s.mean[s.out_slot[r]];
        int best = 0;
        double bd = trk_dist(m, s.pts[0], 4);
        for (int i = 1; i < nf; ++i) { const double d = trk_dist(m, s.pts[i], 4); if (d < bd) { bd = d; best = i; } }
        s.out_det[r] = best;
      }
    }
    __syncthreads();
    if (tid == 0 && stream >= 0) s.out0 = b * 2 * kTrkDet;        // the frame's window
    if (tid == 0 && s.out0 + s.nout > out.capacity) s.ctl[kCtlBroken] = 2;
    __syncthreads();
    if (s.ctl[kCtlBroken]) break;
    // gather (bev/main.py:277-278) and One-Euro smoothing (:280-285 / :262-266), then cam_trans (:169)
    const int nout = s.nout, o0 = s.out0, sig = s.sig;
    for (int r = tid; r < nout; r += blockDim.x) {
      const size_t src = st + s.out_det[r], dst = o0 + r;
      out.batch_ids[dst] = b;
      out.track_ids[dst] = in.show_largest ? 0 : s.meta[s.out_slot[r]][kMetaId];
      out.det[dst] = s.out_det[r];
      out.conf[dst] = in.conf[src];
      oe_rodrigues(in.thetas + src * 72, s.R[r]);
    }
    for (int e = tid; e < nout * 146; e += blockDim.x)
      out.params[(size_t)(o0 + e / 146) * 146 + e % 146] = in.params[(size_t)(st + s.out_det[e / 146]) * 146 + e % 146];
    __syncthreads();
    for (int e = tid; e < nout * kOeCh; e += blockDim.x) {
      const int r = e / kOeCh, c = e % kOeCh;
      const size_t src = st + s.out_det[r], dst = o0 + r;
      const int slot = sig * T + s.out_slot[r];
      const bool seen = g.oe_seen[slot] != 0;
      float x = 0.f, mincut = in.smooth_coeff;
      bool active = true;
      if (c < kOePose) x = s.R[r][c];
      else if (c < kOeBeta) x = in.thetas[src * 72 + 3 + (c - kOePose)];
      else if (c < kOeCam) { active = (c - kOeBeta) < 11; if (active) x = in.betas[src * 11 + (c - kOeBeta)]; mincut = 0.6f; }
      else { x = in.cam[src * 3 + (c - kOeCam)]; mincut = 1.6f; }
      if (!active) continue;
      const size_t o = (size_t)slot * kOeCh + c;
      // tracked mode: pose, betas and cam differentiate against their previous smoothed value (oe_step, aliased)
      const float y = oe_step(x, mincut, 30.f, seen, !in.show_largest && c >= kOePose, &g.oe_raw[o], &g.oe_x[o], &g.oe_dx[o]);
      if (c < kOePose) s.R[r][c] = y;
      else if (c < kOeBeta) out.thetas[dst * 72 + 3 + (c - kOePose)] = y;
      else if (c < kOeCam) out.betas[dst * 11 + (c - kOeBeta)] = y;
      else out.cam[dst * 3 + (c - kOeCam)] = y;
    }
    __syncthreads();
    for (int r = tid; r < nout; r += blockDim.x) {
      const size_t dst = o0 + r;
      float aa[3];
      rotmat_to_aa(s.R[r], aa);                         // smooth_global_rot_matrix, utils.py:191
      out.thetas[dst * 72 + 0] = aa[0]; out.thetas[dst * 72 + 1] = aa[1]; out.thetas[dst * 72 + 2] = aa[2];
      bev_cam_trans_rn(out.cam + dst * 3, out.cam_trans + dst * 3);
      g.oe_seen[sig * T + s.out_slot[r]] = 1;
    }
    __syncthreads();
    if (tid == 0) { s.out0 += nout; s.st = st + s.nf; out.status[2 + b] = nout; }
    __syncthreads();
  }
  __syncthreads();
  for (int i = tid; i < T * 8; i += blockDim.x) g.mean[i] = s.mean[i / 8][i % 8];
  for (int i = tid; i < T * 3; i += blockDim.x) g.S[i] = s.S[i / 3][i % 3];
  for (int i = tid; i < T * kMetaN; i += blockDim.x) g.meta[i] = s.meta[i / kMetaN][i % kMetaN];
  for (int i = tid; i < T; i += blockDim.x) { g.lists[i] = s.tracked[i]; g.lists[T + i] = s.lost[i]; }
  if (tid < kCtlN) g.ctl[tid] = s.ctl[tid];
  if (stream >= 0) {                                    // the failed frame and every later frame of the stream
    if (s.ctl[kCtlBroken])
      for (int f = b + tid; f < in.batch; f += blockDim.x) if (in.sig_slot[f] == stream) out.status[2 + f] = -s.ctl[kCtlBroken];
  } else if (tid == 0) {
    *out.d_count = s.out0;
    out.status[0] = s.ctl[kCtlBroken];
    out.status[1] = s.ctl[kCtlFrame];
  }
}

__global__ void __launch_bounds__(kTrkThreads) bev_track_kernel(TrkDev g, TrkIn in, TrkOut out) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  TrkSmem& s = *reinterpret_cast<TrkSmem*>(smem_raw);
  double* cost = reinterpret_cast<double*>(smem_raw + ((sizeof(TrkSmem) + 15) / 16) * 16);
  bev_track_walk(s, cost, g, in, out, -1);
}

// Stream mode: CTA b steps stream sig_slot[b] when frame b is the stream's first frame in the batch; g.signals = streams.
__global__ void __launch_bounds__(kTrkThreads) bev_track_streams_kernel(TrkDev g, TrkIn in, TrkOut out) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  TrkSmem& s = *reinterpret_cast<TrkSmem*>(smem_raw);
  double* cost = reinterpret_cast<double*>(smem_raw + ((sizeof(TrkSmem) + 15) / 16) * 16);
  const int stream = in.sig_slot[blockIdx.x], T = g.T;
  for (int f = 0; f < (int)blockIdx.x; ++f) if (in.sig_slot[f] == stream) return;
  if (stream < 0 || stream >= g.signals) {              // not a stream of the handle: its frames fail
    for (int f = threadIdx.x; f < in.batch; f += blockDim.x) if (in.sig_slot[f] == stream) out.status[2 + f] = -3;
    return;
  }
  const size_t o = (size_t)stream * T;
  g.mean += o * 8; g.S += o * 3; g.meta += o * kMetaN; g.lists += o * 2; g.ctl += (size_t)stream * kCtlN;
  g.oe_raw += o * kOeCh; g.oe_x += o * kOeCh; g.oe_dx += o * kOeCh; g.oe_seen += o;
  g.signals = 1;
  bev_track_walk(s, cost, g, in, out, stream);
}

// Stream mode, after bev_track_streams_kernel (one CTA): moves every frame's rows from its window to the end of the
// previous frames' rows, in frame order.  A frame's rows move down by d = window start - destination; copying them in
// chunks of at most d rows never overwrites a row before it is read.  Writes *d_count and status[0] = the frames whose
// stream failed, status[1] = 0.
template <typename V>
__device__ __forceinline__ void trk_move_rows(V* p, int w, int dst, int src, int n) {
  for (int e = threadIdx.x; e < n * w; e += blockDim.x) p[(size_t)dst * w + e] = p[(size_t)src * w + e];
}

__global__ void __launch_bounds__(1024) bev_track_compact_kernel(TrkOut out, int batch) {
  int total = 0, failed = 0;
  for (int b = 0; b < batch; ++b) {
    const int n = out.status[2 + b], src = b * 2 * kTrkDet;
    failed += n < 0;
    if (n <= 0) continue;
    const int d = src - total;
    for (int r0 = 0; r0 < n && d > 0; r0 += d) {
      const int c = min(d, n - r0), from = src + r0, to = total + r0;
      trk_move_rows(out.batch_ids, 1, to, from, c);
      trk_move_rows(out.track_ids, 1, to, from, c);
      trk_move_rows(out.det, 1, to, from, c);
      trk_move_rows(out.conf, 1, to, from, c);
      trk_move_rows(out.thetas, 72, to, from, c);
      trk_move_rows(out.betas, 11, to, from, c);
      trk_move_rows(out.cam, 3, to, from, c);
      trk_move_rows(out.cam_trans, 3, to, from, c);
      trk_move_rows(out.params, 146, to, from, c);
      __syncthreads();
    }
    total += n;
  }
  if (threadIdx.x == 0) { *out.d_count = total; out.status[0] = failed; out.status[1] = 0; }
}

constexpr size_t kTrkSmem = ((sizeof(TrkSmem) + 15) / 16) * 16 + sizeof(double) * kTrkMax * kTrkDet;

}  // namespace b200romp

using namespace b200romp;

struct b200romp_bev_tracker {
  int device = 0;
  int streams = 0;     // 0: one tracker and max_signals filter sets; > 0: that many independent trackers (stream mode)
  TrkDev d{};
};

static b200romp_bev_tracker* bev_tracker_new(int device, int max_tracks, int filter_sets, int streams) {
  b200romp_bev_tracker* t = new b200romp_bev_tracker();
  t->device = device;
  t->streams = streams;
  TrkDev& d = t->d;
  d.T = max_tracks; d.signals = filter_sets;
  const size_t trackers = streams > 0 ? streams : 1, T = trackers * max_tracks;
  const size_t slots = (size_t)filter_sets * max_tracks, nf = slots * kOeCh * sizeof(float);
  bool ok = cudaMalloc(&d.mean, T * 8 * sizeof(double)) == cudaSuccess &&
            cudaMalloc(&d.S, T * 3 * sizeof(double)) == cudaSuccess &&
            cudaMalloc(&d.meta, T * kMetaN * sizeof(int)) == cudaSuccess &&
            cudaMalloc(&d.lists, 2 * T * sizeof(int)) == cudaSuccess &&
            cudaMalloc(&d.ctl, trackers * kCtlN * sizeof(int)) == cudaSuccess &&
            cudaMalloc(&d.oe_raw, nf) == cudaSuccess && cudaMalloc(&d.oe_x, nf) == cudaSuccess && cudaMalloc(&d.oe_dx, nf) == cudaSuccess &&
            cudaMalloc(&d.oe_seen, slots * sizeof(int)) == cudaSuccess &&
            cudaFuncSetAttribute(bev_track_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kTrkSmem) == cudaSuccess &&
            cudaFuncSetAttribute(bev_track_streams_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kTrkSmem) == cudaSuccess &&
            cudaMemset(d.mean, 0, T * 8 * sizeof(double)) == cudaSuccess &&
            cudaMemset(d.S, 0, T * 3 * sizeof(double)) == cudaSuccess &&
            cudaMemset(d.meta, 0, T * kMetaN * sizeof(int)) == cudaSuccess &&
            cudaMemset(d.lists, 0, 2 * T * sizeof(int)) == cudaSuccess &&
            cudaMemset(d.ctl, 0, trackers * kCtlN * sizeof(int)) == cudaSuccess &&
            cudaMemset(d.oe_seen, 0, slots * sizeof(int)) == cudaSuccess;
  if (!ok) {
    set_error("bev_tracker_create: allocation failed");
    b200romp_bev_tracker_destroy(t);
    return nullptr;
  }
  return t;
}

extern "C" {

b200romp_bev_tracker* b200romp_bev_tracker_create(int device, int max_tracks, int max_signals) {
  if (max_tracks <= 0 || max_tracks > kTrkMax || max_signals <= 0 || cudaSetDevice(device) != cudaSuccess) {
    set_error("bev_tracker_create: bad arguments (1 <= max_tracks <= %d, max_signals >= 1) / no CUDA device", kTrkMax);
    return nullptr;
  }
  return bev_tracker_new(device, max_tracks, max_signals, 0);
}

b200romp_bev_tracker* b200romp_bev_tracker_create_streams(int device, int max_tracks, int streams) {
  if (max_tracks <= 0 || max_tracks > kTrkMax || streams <= 0 || streams > B200ROMP_MAX_VIDEO_STREAMS ||
      cudaSetDevice(device) != cudaSuccess) {
    set_error("bev_tracker_create_streams: bad arguments (1 <= max_tracks <= %d, 1 <= streams <= %d) / no CUDA device", kTrkMax,
              B200ROMP_MAX_VIDEO_STREAMS);
    return nullptr;
  }
  return bev_tracker_new(device, max_tracks, streams, streams);
}

void b200romp_bev_tracker_destroy(b200romp_bev_tracker* t) {
  if (!t) return;
  cudaSetDevice(t->device);
  TrkDev& d = t->d;
  cudaFree(d.mean); cudaFree(d.S); cudaFree(d.meta); cudaFree(d.lists); cudaFree(d.ctl);
  cudaFree(d.oe_raw); cudaFree(d.oe_x); cudaFree(d.oe_dx); cudaFree(d.oe_seen);
  delete t;
}

int b200romp_bev_tracker_reset(b200romp_bev_tracker* t, int signal, b200romp_stream stream_) {
  B2R_REQUIRE(t && signal >= -1 && signal < t->d.signals, "bev_tracker_reset: bad signal");
  B2R_CUDA_OK(cudaSetDevice(t->device));
  cudaStream_t stream = (cudaStream_t)stream_;
  const TrkDev& d = t->d;
  if (signal < 0) {
    const size_t trackers = t->streams > 0 ? t->streams : 1;
    B2R_CUDA_OK(cudaMemsetAsync(d.meta, 0, trackers * d.T * kMetaN * sizeof(int), stream));
    B2R_CUDA_OK(cudaMemsetAsync(d.ctl, 0, trackers * kCtlN * sizeof(int), stream));
    B2R_CUDA_OK(cudaMemsetAsync(d.oe_seen, 0, (size_t)d.signals * d.T * sizeof(int), stream));
  } else {
    if (t->streams > 0) {                              // the stream's tracker: no tracks, frame_id 0, ids from 1
      B2R_CUDA_OK(cudaMemsetAsync(d.meta + (size_t)signal * d.T * kMetaN, 0, d.T * kMetaN * sizeof(int), stream));
      B2R_CUDA_OK(cudaMemsetAsync(d.ctl + (size_t)signal * kCtlN, 0, kCtlN * sizeof(int), stream));
    }
    B2R_CUDA_OK(cudaMemsetAsync(d.oe_seen + (size_t)signal * d.T, 0, d.T * sizeof(int), stream));
  }
  return B200ROMP_OK;
}

int b200romp_bev_track_step(b200romp_bev_tracker* t, int batch, int capacity, const int* d_count, const long long* batch_ids,
                            const float* conf, const float* cam, const float* cam_trans, const float* thetas, const float* betas,
                            const float* params_pred, const int* signal_slot, int show_largest, float smooth_coeff, int out_capacity,
                            int* d_out_count, long long* out_batch_ids, int* out_track_ids, int* out_det, float* out_thetas,
                            float* out_betas, float* out_cam, float* out_cam_trans, float* out_params_pred, float* out_conf,
                            int* d_status, b200romp_stream stream_) {
  B2R_REQUIRE(t && batch > 0 && capacity > 0 && d_count && batch_ids && conf && cam && cam_trans && thetas && betas && params_pred &&
                  signal_slot && out_capacity > 0 && d_out_count && out_batch_ids && out_track_ids && out_det && out_thetas &&
                  out_betas && out_cam && out_cam_trans && out_params_pred && out_conf && d_status,
              "bev_track_step: bad arguments");
  B2R_CUDA_OK(cudaSetDevice(t->device));
  TrkIn in{d_count, batch_ids, conf, cam, cam_trans, thetas, betas, params_pred, signal_slot, batch, capacity, show_largest, smooth_coeff};
  TrkOut out{out_capacity, d_out_count, out_batch_ids, out_track_ids, out_det, out_thetas, out_betas, out_cam, out_cam_trans,
             out_params_pred, out_conf, d_status};
  if (t->streams > 0) {
    bev_track_streams_kernel<<<batch, kTrkThreads, kTrkSmem, (cudaStream_t)stream_>>>(t->d, in, out);
    B2R_CUDA_OK(cudaGetLastError());
    bev_track_compact_kernel<<<1, 1024, 0, (cudaStream_t)stream_>>>(out, batch);
  } else {
    bev_track_kernel<<<1, kTrkThreads, kTrkSmem, (cudaStream_t)stream_>>>(t->d, in, out);
  }
  B2R_CUDA_OK(cudaGetLastError());
  return B200ROMP_OK;
}

}  // extern "C"
