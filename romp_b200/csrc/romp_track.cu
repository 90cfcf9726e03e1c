// ROMP's video mode for batches (ROMP.forward_video, --temporal_optimize): the association of ROMP.forward's temporal path
// (romp_b200/temporal.py: TemporalState.assign with NearestCenterTracker, the stand-in for the reference's norfair tracker,
// simple_romp/romp/main.py:117-157) and its One-Euro smoothing (temporal.cu's recurrences), as ONE kernel per batch between
// b200romp_parse and SMPL.  One CTA walks the batch's frames in order, because every frame's association depends on the
// state the previous frame left; threads parallelise over tracks (argmin, ageing, compaction) and over row channels
// (smoothing).  The tracker state of every signal and the filter state of every slot stay in device memory.
// Stream mode (a streams handle): one signal block per stream index, no registration by code; one CTA per stream present
// in the batch walks that stream's frames with the same per-frame step (romp_track_walk).
//
// Per frame with at least one detection (a frame with nobody does nothing, like forward):
//   signal: a new signal code takes the lowest free block of 64 filter slots and resets all of them; with every block in
//   use it first evicts the signal registered earliest (FIFO by first registration).  A returning signal starts afresh.
//   --show_largest: no tracker; the row argmax(cam[:,0]) (first on ties) uses the block's base slot, untracked recurrence.
//   tracked: NearestCenterTracker.update on the points cam[:,[2,1]] * 512 (fp32 product, distances in fp64): detections in
//   row order, each takes the live track at the smallest distance strictly below 200 (the earliest created on ties) and
//   moves it at once, else it creates a track with the next id; then every unmatched track ages and is dropped once its
//   age exceeds 30.  Slots of dropped tracks are freed; a track without a slot takes the lowest free slot of its block
//   (reset), in detection order, or stays unsmoothed (-1) when none is free; of two rows on one slot the first keeps it.
//   Smoothing with the tracked recurrence.
//
// Track table size: a frame has at most 64 detections and a track unmatched for 31 stepped frames of its signal is gone,
// so at the start of a frame every live track was matched (or created) in one of the signal's last 31 stepped frames: at
// most 31 x 64 tracks, and 32 x 64 = 2048 counting the ones the current frame creates.  kRtTracks is that bound, so the
// step never runs out of table.
#include "common.cuh"
#include "rot6d.cuh"
#include "one_euro.cuh"
#include <limits.h>

namespace b200romp {

constexpr int kRtDet = 64;                         // detections per frame (MAX_PERSON)
constexpr int kRtBlock = 64;                       // filter slots per signal (temporal.py MAX_TRACKS_PER_SIGNAL)
constexpr int kRtMaxAge = 30;                      // NearestCenterTracker max_age
constexpr int kRtTracks = (kRtMaxAge + 2) * kRtDet;  // 2048, see the bound above
constexpr int kRtMaxSignals = 16;
constexpr int kRtThreads = 512;
constexpr int kRtPer = kRtTracks / kRtThreads;     // track entries per thread in the compaction
constexpr int kRtBetas = 10;
constexpr double kRtThr = 200.0;                   // distance_threshold
enum { kSigCode = 0, kSigSeq, kSigN, kSigNextId, kSigFields };   // kSigSeq = 0: block free

struct RtDev {
  double* pt;               // [signals][kRtTracks][2] track points, creation order
  int* id;                  // [signals][kRtTracks]
  int* age;                 // [signals][kRtTracks]
  int* slot;                // [signals][kRtTracks] absolute filter slot or -1
  int* sig;                 // [signals][kSigFields]; block index = signal table index
  unsigned long long* mask; // [signals] slots of the block held by a live track
  int* reg;                 // [1] registrations so far
  float *oe_raw, *oe_x, *oe_dx;   // [signals * 64][kOeCh]
  int* oe_seen;             // [signals * 64]
  int signals;
};

struct RtSmem {
  double pt[kRtTracks][2];
  int id[kRtTracks], age[kRtTracks], slot[kRtTracks];
  unsigned char matched[kRtTracks];
  int sig[kRtMaxSignals][kSigFields];
  unsigned long long mask[kRtMaxSignals];
  int reg, loaded, blk, st, nf, nrows, out0;
  double dpt[kRtDet][2];
  int det_e[kRtDet], row_id[kRtDet], row_slot[kRtDet], row_src[kRtDet], row_dst[kRtDet];
  float R[kRtDet][9];
  double red_d[kRtThreads / 32];
  int red_e[kRtThreads / 32], warp_sum[kRtThreads / 32];
};

struct RtIn {
  const int* d_count; const long long* batch_ids; const float *cam, *thetas, *betas; const int* sig_code;
  int batch, capacity, show_largest; float smooth_coeff, freq;
};
struct RtOut {
  int* d_count; long long* batch_ids; float *thetas, *betas, *cam; int *slot, *track_ids;
};

__device__ __forceinline__ double rt_dist(const double* q, const double* p) {
  const double dx = __dsub_rn(p[0], q[0]), dy = __dsub_rn(p[1], q[1]);    // np.linalg.norm(p - q), no contraction
  return sqrt(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)));
}

__device__ void rt_table_io(RtSmem& s, const RtDev& g, int blk, int n, bool load) {
  const size_t o = (size_t)blk * kRtTracks;
  for (int e = threadIdx.x; e < n; e += blockDim.x) {
    if (load) {
      s.pt[e][0] = g.pt[(o + e) * 2]; s.pt[e][1] = g.pt[(o + e) * 2 + 1];
      s.id[e] = g.id[o + e]; s.age[e] = g.age[o + e]; s.slot[e] = g.slot[o + e]; s.matched[e] = 0;
    } else {
      g.pt[(o + e) * 2] = s.pt[e][0]; g.pt[(o + e) * 2 + 1] = s.pt[e][1];
      g.id[o + e] = s.id[e]; g.age[o + e] = s.age[e]; g.slot[o + e] = s.slot[e];
    }
  }
}

// one detection of NearestCenterTracker.update: argmin over the live tracks of (distance < 200, creation order)
__device__ void rt_associate(RtSmem& s, int i) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, n = s.sig[s.blk][kSigN];
  double bd = kRtThr;
  int be = INT_MAX;
  for (int e = tid; e < n; e += blockDim.x) {
    const double d = rt_dist(s.pt[e], s.dpt[i]);
    if (d < bd) { bd = d; be = e; }
  }
  for (int off = 16; off; off >>= 1) {
    const double od = __shfl_xor_sync(0xffffffffu, bd, off);
    const int oe = __shfl_xor_sync(0xffffffffu, be, off);
    if (od < bd || (od == bd && oe < be)) { bd = od; be = oe; }
  }
  if (lane == 0) { s.red_d[warp] = bd; s.red_e[warp] = be; }
  __syncthreads();
  if (tid == 0) {
    for (int w = 1; w < (int)(blockDim.x >> 5); ++w)
      if (s.red_d[w] < bd || (s.red_d[w] == bd && s.red_e[w] < be)) { bd = s.red_d[w]; be = s.red_e[w]; }
    int* sg = s.sig[s.blk];
    if (be == INT_MAX) {                          // a new track, appended: the table stays in creation (= id) order
      be = sg[kSigN]++;
      s.id[be] = sg[kSigNextId]++;
      s.slot[be] = -1;
    }
    s.pt[be][0] = s.dpt[i][0]; s.pt[be][1] = s.dpt[i][1];
    s.age[be] = 0; s.matched[be] = 1;
    s.det_e[i] = be; s.row_id[i] = s.id[be];
  }
  __syncthreads();
}

// ageing, slot release and stable compaction of the live tracks (all threads)
__device__ void rt_age_and_compact(RtSmem& s) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, n = s.sig[s.blk][kSigN], base = s.blk * kRtBlock;
  double pt[kRtPer][2];
  int id[kRtPer], age[kRtPer], slot[kRtPer], keep = 0;
  bool live[kRtPer];
#pragma unroll
  for (int k = 0; k < kRtPer; ++k) {
    const int e = tid * kRtPer + k;
    live[k] = false;
    if (e < n) {
      pt[k][0] = s.pt[e][0]; pt[k][1] = s.pt[e][1]; id[k] = s.id[e]; slot[k] = s.slot[e]; age[k] = s.age[e];
      if (!s.matched[e]) ++age[k];
      live[k] = age[k] <= kRtMaxAge;
      keep += live[k];
    }
  }
  int incl = keep;
  for (int off = 1; off < 32; off <<= 1) {
    const int v = __shfl_up_sync(0xffffffffu, incl, off);
    if (lane >= off) incl += v;
  }
  if (lane == 31) s.warp_sum[warp] = incl;
  __syncthreads();                                  // every entry is in registers: the table may be rewritten
  int pos = incl - keep, total = 0;
  for (int w = 0; w < (int)(blockDim.x >> 5); ++w) { if (w < warp) pos += s.warp_sum[w]; total += s.warp_sum[w]; }
  unsigned long long freed = 0;
#pragma unroll
  for (int k = 0; k < kRtPer; ++k) {
    const int e = tid * kRtPer + k;
    if (e >= n) continue;
    if (live[k]) {
      s.pt[pos][0] = pt[k][0]; s.pt[pos][1] = pt[k][1]; s.id[pos] = id[k]; s.age[pos] = age[k]; s.slot[pos] = slot[k];
      s.matched[pos] = 0;
      ++pos;
    } else if (slot[k] >= 0) {
      freed |= 1ull << (slot[k] - base);
    }
  }
  if (freed) atomicAnd(&s.mask[s.blk], ~freed);
  __syncthreads();
  if (tid == 0) s.sig[s.blk][kSigN] = total;
  __syncthreads();
}

// frames with at least one of the rows [0, n) (grouped by frame); called by every thread of the CTA
__device__ int rt_frames_with_rows(const long long* batch_ids, int n) {
  int c = 0;
  for (int r0 = 0; r0 < n; r0 += blockDim.x) {
    const int r = r0 + threadIdx.x;
    c += __syncthreads_count(r < n && (r == 0 || batch_ids[r] != batch_ids[r - 1]));
  }
  return c;
}

// The walk of the batch's frames in order.  stream < 0: every frame, with the signal registration above, and the batch's
// output count (and the tracked mode's batch ids) written at the end.  stream >= 0 (g offset to that stream's state, one
// signal block whose code is the stream index): only the frames with sig_code[b] == stream; --show_largest writes frame
// b's row after the frames before it that have rows.
__device__ void romp_track_walk(RtSmem& s, const RtDev& g, const RtIn& in, const RtOut& out, int stream) {
  const int tid = threadIdx.x;
  for (int i = tid; i < g.signals * kSigFields; i += blockDim.x) s.sig[i / kSigFields][i % kSigFields] = g.sig[i];
  for (int i = tid; i < g.signals; i += blockDim.x) s.mask[i] = g.mask[i];
  if (tid == 0) { s.reg = *g.reg; s.loaded = -1; s.st = 0; s.out0 = 0; }
  __syncthreads();
  const int N = min(*in.d_count, in.capacity);
  const bool tracked = !in.show_largest;
  for (int b = 0; b < in.batch; ++b) {
    if (stream >= 0 && in.sig_code[b] != stream) continue;     // another stream's frame
    if (tid == 0) {                                 // rows of frame b (the parse groups them by frame, in frame order)
      int st = s.st;
      while (st < N && in.batch_ids[st] < b) ++st;
      int e = st;
      while (e < N && in.batch_ids[e] == b) ++e;
      s.st = st; s.nf = min(e - st, kRtDet);
    }
    __syncthreads();
    const int st = s.st, nf = s.nf;
    if (nf == 0) { __syncthreads(); continue; }     // forward returns before TemporalState.assign
    if (stream >= 0 && !tracked) {                  // row of frame b = the frames with rows before it
      const int c = rt_frames_with_rows(in.batch_ids, st);
      if (tid == 0) s.out0 = c;
    }
    int fresh = 0;
    if (tid == 0) {                                 // TemporalState.assign: the signal's block
      const int code = in.sig_code[b];
      int blk = -1, used = 0, oldest = -1;
      for (int q = 0; q < g.signals; ++q) {
        if (!s.sig[q][kSigSeq]) continue;
        ++used;
        if (s.sig[q][kSigCode] == code) blk = q;
        if (oldest < 0 || s.sig[q][kSigSeq] < s.sig[oldest][kSigSeq]) oldest = q;
      }
      if (blk < 0) {
        if (used >= g.signals) s.sig[oldest][kSigSeq] = 0;      // evict the earliest registration
        blk = 0;
        while (s.sig[blk][kSigSeq]) ++blk;
        s.sig[blk][kSigCode] = code; s.sig[blk][kSigSeq] = ++s.reg; s.sig[blk][kSigN] = 0; s.sig[blk][kSigNextId] = 1;
        s.mask[blk] = 0;
        fresh = 1;
      }
      s.blk = blk;
      s.nrows = fresh;                              // broadcast through shared memory below
    }
    __syncthreads();
    const int blk = s.blk, base = blk * kRtBlock;
    fresh = s.nrows;
    if (fresh && tid < kRtBlock) g.oe_seen[base + tid] = 0;           // every slot of a new signal's block
    if (tracked && blk != s.loaded) {               // bring the signal's track table into shared memory
      if (s.loaded >= 0) rt_table_io(s, g, s.loaded, s.sig[s.loaded][kSigN], false);
      rt_table_io(s, g, blk, s.sig[blk][kSigN], true);
    }
    __syncthreads();
    if (tid == 0) s.loaded = tracked ? blk : -1;
    if (!tracked) {
      if (tid == 0) {                               // argmax(cam[:,0]), the first on ties
        int best = 0;
        for (int i = 1; i < nf; ++i) if (in.cam[(size_t)(st + i) * 3] > in.cam[(size_t)(st + best) * 3]) best = i;
        for (int i = 0; i < nf; ++i) { out.slot[st + i] = i == best ? base : -1; out.track_ids[st + i] = 0; }
        s.nrows = 1; s.row_src[0] = st + best; s.row_dst[0] = s.out0; s.row_slot[0] = base;
        out.batch_ids[s.out0] = b;
      }
    } else {
      if (tid < nf) {                               // cam[:,[2,1]] * 512 in fp32, then fp64
        s.dpt[tid][0] = (double)__fmul_rn(in.cam[(size_t)(st + tid) * 3 + 2], 512.f);
        s.dpt[tid][1] = (double)__fmul_rn(in.cam[(size_t)(st + tid) * 3 + 1], 512.f);
      }
      __syncthreads();
      for (int i = 0; i < nf; ++i) rt_associate(s, i);
      // a track dropped now releases its slot before this frame's new tracks claim one; the detections' tracks are live
      rt_age_and_compact(s);
      if (tid == 0) {
        // compaction moved the entries: find each detection's track again by id (ids increase along the table)
        for (int i = 0; i < nf; ++i) {
          int lo = 0, hi = s.sig[blk][kSigN] - 1;
          while (lo < hi) { const int m = (lo + hi) >> 1; if (s.id[m] < s.row_id[i]) lo = m + 1; else hi = m; }
          s.det_e[i] = lo;
        }
        unsigned long long held = 0;
        for (int i = 0; i < nf; ++i) {
          const int e = s.det_e[i];
          if (s.slot[e] < 0) {
            const unsigned long long free = ~s.mask[blk];
            if (free) {
              const int k = __ffsll((long long)free) - 1;
              s.mask[blk] |= 1ull << k;
              s.slot[e] = base + k;
              g.oe_seen[base + k] = 0;              // a newly claimed slot starts fresh
            }
          }
          int sl = s.slot[e];
          if (sl >= 0) {
            if (held >> (sl - base) & 1ull) sl = -1;                  // a second row on one track stays unsmoothed
            else held |= 1ull << (sl - base);
          }
          s.row_slot[i] = sl; s.row_src[i] = st + i; s.row_dst[i] = st + i;
          out.slot[st + i] = sl; out.track_ids[st + i] = s.row_id[i];
        }
        s.nrows = nf;
      }
    }
    __syncthreads();
    // One-Euro smoothing of the frame's rows (temporal.cu one_euro_kernel, row by row)
    const int nrows = s.nrows;
    for (int r = tid; r < nrows; r += blockDim.x)
      if (s.row_slot[r] >= 0) oe_rodrigues(in.thetas + (size_t)s.row_src[r] * 72, s.R[r]);
    __syncthreads();
    for (int e = tid; e < nrows * kOeCh; e += blockDim.x) {
      const int r = e / kOeCh, c = e % kOeCh, sl = s.row_slot[r];
      const size_t src = s.row_src[r], dst = s.row_dst[r];
      float x = 0.f, mincut = in.smooth_coeff;
      bool active = true;
      if (c < kOePose) x = s.R[r][c];
      else if (c < kOeBeta) x = in.thetas[src * 72 + 3 + (c - kOePose)];
      else if (c < kOeCam) { active = (c - kOeBeta) < kRtBetas; if (active) x = in.betas[src * kRtBetas + (c - kOeBeta)]; mincut = 0.6f; }
      else { x = in.cam[src * 3 + (c - kOeCam)]; mincut = 1.6f; }
      if (!active) continue;
      float y = x;
      if (sl >= 0) {
        const size_t o = (size_t)sl * kOeCh + c;
        y = oe_step(x, mincut, in.freq, g.oe_seen[sl] != 0, tracked && c >= kOePose, &g.oe_raw[o], &g.oe_x[o], &g.oe_dx[o]);
      }
      if (c < kOePose) s.R[r][c] = y;
      else if (c < kOeBeta) out.thetas[dst * 72 + 3 + (c - kOePose)] = y;
      else if (c < kOeCam) out.betas[dst * kRtBetas + (c - kOeBeta)] = y;
      else out.cam[dst * 3 + (c - kOeCam)] = y;
    }
    __syncthreads();
    for (int r = tid; r < nrows; r += blockDim.x) {
      const size_t src = s.row_src[r], dst = s.row_dst[r];
      const int sl = s.row_slot[r];
      if (sl >= 0) {
        float aa[3];
        rotmat_to_aa(s.R[r], aa);
        out.thetas[dst * 72 + 0] = aa[0]; out.thetas[dst * 72 + 1] = aa[1]; out.thetas[dst * 72 + 2] = aa[2];
        g.oe_seen[sl] = 1;
      } else {
        for (int k = 0; k < 3; ++k) out.thetas[dst * 72 + k] = in.thetas[src * 72 + k];
      }
    }
    __syncthreads();
    if (tid == 0) { s.st = st + nf; if (!tracked) ++s.out0; }
    __syncthreads();
  }
  if (s.loaded >= 0) rt_table_io(s, g, s.loaded, s.sig[s.loaded][kSigN], false);
  for (int i = tid; i < g.signals * kSigFields; i += blockDim.x) g.sig[i] = s.sig[i / kSigFields][i % kSigFields];
  for (int i = tid; i < g.signals; i += blockDim.x) g.mask[i] = s.mask[i];
  if (tid == 0) *g.reg = s.reg;
  if (stream >= 0) return;
  if (tracked) for (int r = tid; r < N; r += blockDim.x) out.batch_ids[r] = in.batch_ids[r];
  if (tid == 0) *out.d_count = tracked ? N : s.out0;
}

__global__ void __launch_bounds__(kRtThreads, 1) romp_track_kernel(RtDev g, RtIn in, RtOut out) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  romp_track_walk(*reinterpret_cast<RtSmem*>(smem_raw), g, in, out, -1);
}

// Stream mode: CTA b steps stream sig_code[b] when frame b is the stream's first frame in the batch; g.signals = streams.
// CTA 0 also writes the batch's output count (and the tracked mode's batch ids).
__global__ void __launch_bounds__(kRtThreads, 1) romp_track_streams_kernel(RtDev g, RtIn in, RtOut out) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int stream = in.sig_code[blockIdx.x];
  for (int f = 0; f < (int)blockIdx.x; ++f) if (in.sig_code[f] == stream) return;
  if (blockIdx.x == 0) {
    const int N = min(*in.d_count, in.capacity);
    if (!in.show_largest) for (int r = threadIdx.x; r < N; r += blockDim.x) out.batch_ids[r] = in.batch_ids[r];
    const int c = in.show_largest ? rt_frames_with_rows(in.batch_ids, N) : N;
    if (threadIdx.x == 0) *out.d_count = c;
  }
  if (stream < 0 || stream >= g.signals) return;      // not a stream of the handle: its frames are left as they are
  const size_t o = (size_t)stream * kRtTracks, f = (size_t)stream * kRtBlock;
  g.pt += o * 2; g.id += o; g.age += o; g.slot += o; g.sig += (size_t)stream * kSigFields; g.mask += stream; g.reg += stream;
  g.oe_raw += f * kOeCh; g.oe_x += f * kOeCh; g.oe_dx += f * kOeCh; g.oe_seen += f;
  g.signals = 1;
  romp_track_walk(*reinterpret_cast<RtSmem*>(smem_raw), g, in, out, stream);
}

constexpr size_t kRtSmem = sizeof(RtSmem);

}  // namespace b200romp

using namespace b200romp;

struct b200romp_romp_tracker {
  int device = 0;
  int streams = 0;     // 0: max_signals signals registered by code; > 0: that many independent streams (stream mode)
  RtDev d{};
};

static b200romp_romp_tracker* romp_tracker_new(int device, int signals, int streams) {
  b200romp_romp_tracker* t = new b200romp_romp_tracker();
  t->device = device;
  t->streams = streams;
  RtDev& d = t->d;
  d.signals = signals;
  const size_t T = (size_t)signals * kRtTracks, slots = (size_t)signals * kRtBlock, nf = slots * kOeCh * sizeof(float);
  const size_t regs = streams > 0 ? streams : 1;     // registration counters: one per stream
  bool ok = cudaMalloc(&d.pt, T * 2 * sizeof(double)) == cudaSuccess && cudaMalloc(&d.id, T * sizeof(int)) == cudaSuccess &&
            cudaMalloc(&d.age, T * sizeof(int)) == cudaSuccess && cudaMalloc(&d.slot, T * sizeof(int)) == cudaSuccess &&
            cudaMalloc(&d.sig, signals * kSigFields * sizeof(int)) == cudaSuccess &&
            cudaMalloc(&d.mask, signals * sizeof(unsigned long long)) == cudaSuccess &&
            cudaMalloc(&d.reg, regs * sizeof(int)) == cudaSuccess &&
            cudaMalloc(&d.oe_raw, nf) == cudaSuccess && cudaMalloc(&d.oe_x, nf) == cudaSuccess && cudaMalloc(&d.oe_dx, nf) == cudaSuccess &&
            cudaMalloc(&d.oe_seen, slots * sizeof(int)) == cudaSuccess &&
            cudaFuncSetAttribute(romp_track_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kRtSmem) == cudaSuccess &&
            cudaFuncSetAttribute(romp_track_streams_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kRtSmem) == cudaSuccess &&
            cudaMemset(d.sig, 0, signals * kSigFields * sizeof(int)) == cudaSuccess &&
            cudaMemset(d.mask, 0, signals * sizeof(unsigned long long)) == cudaSuccess &&
            cudaMemset(d.reg, 0, regs * sizeof(int)) == cudaSuccess && cudaMemset(d.oe_seen, 0, slots * sizeof(int)) == cudaSuccess;
  if (!ok) {
    set_error("romp_tracker_create: allocation failed");
    b200romp_romp_tracker_destroy(t);
    return nullptr;
  }
  return t;
}

extern "C" {

b200romp_romp_tracker* b200romp_romp_tracker_create(int device, int max_signals) {
  if (max_signals <= 0 || max_signals > kRtMaxSignals || cudaSetDevice(device) != cudaSuccess) {
    set_error("romp_tracker_create: bad arguments (1 <= max_signals <= %d) / no CUDA device", kRtMaxSignals);
    return nullptr;
  }
  return romp_tracker_new(device, max_signals, 0);
}

b200romp_romp_tracker* b200romp_romp_tracker_create_streams(int device, int streams) {
  if (streams <= 0 || streams > B200ROMP_MAX_VIDEO_STREAMS || cudaSetDevice(device) != cudaSuccess) {
    set_error("romp_tracker_create_streams: bad arguments (1 <= streams <= %d) / no CUDA device", B200ROMP_MAX_VIDEO_STREAMS);
    return nullptr;
  }
  return romp_tracker_new(device, streams, streams);
}

void b200romp_romp_tracker_destroy(b200romp_romp_tracker* t) {
  if (!t) return;
  cudaSetDevice(t->device);
  RtDev& d = t->d;
  cudaFree(d.pt); cudaFree(d.id); cudaFree(d.age); cudaFree(d.slot); cudaFree(d.sig); cudaFree(d.mask); cudaFree(d.reg);
  cudaFree(d.oe_raw); cudaFree(d.oe_x); cudaFree(d.oe_dx); cudaFree(d.oe_seen);
  delete t;
}

int b200romp_romp_tracker_reset(b200romp_romp_tracker* t, b200romp_stream stream_) {
  B2R_REQUIRE(t, "romp_tracker_reset: bad arguments");
  B2R_CUDA_OK(cudaSetDevice(t->device));
  cudaStream_t stream = (cudaStream_t)stream_;
  const RtDev& d = t->d;
  B2R_CUDA_OK(cudaMemsetAsync(d.sig, 0, d.signals * kSigFields * sizeof(int), stream));   // every block free
  B2R_CUDA_OK(cudaMemsetAsync(d.mask, 0, d.signals * sizeof(unsigned long long), stream));
  B2R_CUDA_OK(cudaMemsetAsync(d.reg, 0, (t->streams > 0 ? t->streams : 1) * sizeof(int), stream));
  B2R_CUDA_OK(cudaMemsetAsync(d.oe_seen, 0, (size_t)d.signals * kRtBlock * sizeof(int), stream));
  return B200ROMP_OK;
}

int b200romp_romp_tracker_reset_stream(b200romp_romp_tracker* t, int s, b200romp_stream stream_) {
  B2R_REQUIRE(t && t->streams > 0 && s >= 0 && s < t->streams, "romp_tracker_reset_stream: not a stream of a streams handle");
  B2R_CUDA_OK(cudaSetDevice(t->device));
  cudaStream_t stream = (cudaStream_t)stream_;
  const RtDev& d = t->d;
  // a free block: the stream's next frame with rows registers it afresh (no tracks, ids from 1, every filter slot reset)
  B2R_CUDA_OK(cudaMemsetAsync(d.sig + (size_t)s * kSigFields, 0, kSigFields * sizeof(int), stream));
  B2R_CUDA_OK(cudaMemsetAsync(d.mask + s, 0, sizeof(unsigned long long), stream));
  return B200ROMP_OK;
}

int b200romp_romp_track_step(b200romp_romp_tracker* t, int batch, int capacity, const int* d_count, const long long* batch_ids,
                             const float* cam, const float* thetas, const float* betas, const int* signal_code, int show_largest,
                             float smooth_coeff, float freq, int* d_out_count, long long* out_batch_ids, float* out_thetas,
                             float* out_betas, float* out_cam, int* out_slot, int* out_track_ids, b200romp_stream stream_) {
  B2R_REQUIRE(t && batch > 0 && capacity > 0 && d_count && batch_ids && cam && thetas && betas && signal_code && d_out_count &&
                  out_batch_ids && out_thetas && out_betas && out_cam && out_slot && out_track_ids,
              "romp_track_step: bad arguments");
  B2R_CUDA_OK(cudaSetDevice(t->device));
  RtIn in{d_count, batch_ids, cam, thetas, betas, signal_code, batch, capacity, show_largest, smooth_coeff, freq};
  RtOut out{d_out_count, out_batch_ids, out_thetas, out_betas, out_cam, out_slot, out_track_ids};
  if (t->streams > 0)
    romp_track_streams_kernel<<<batch, kRtThreads, kRtSmem, (cudaStream_t)stream_>>>(t->d, in, out);
  else
    romp_track_kernel<<<1, kRtThreads, kRtSmem, (cudaStream_t)stream_>>>(t->d, in, out);
  B2R_CUDA_OK(cudaGetLastError());
  return B200ROMP_OK;
}

}  // extern "C"
