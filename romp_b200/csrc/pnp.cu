// cam_trans by RANSAC around EPnP, on the device: ``--cam_trans epnp``.
//
// Replaces, per person, simple_romp/romp: estimate_translation utils.py:391-436 (the validity mask of the 24 SMPL joints
// against their weak-perspective projection, INVALID_TRANS below 4 valid joints) -> estimate_translation_cv2 :331-345,
// i.e. cv2.solvePnPRansac(flags=SOLVEPNP_EPNP, reprojectionError=20, iterationsCount=100) with K = [[443.4,0,256],
// [0,443.4,256],[0,0,1]] (post_parser.py:96-101).  The RANSAC loop is OpenCV's (RANSACPointSetRegistrator::run): its
// RNG seeded with (uint64)-1, 5-point subsets drawn without repeats, a model replacing the best when its inlier count
// exceeds max(best, 4), the iteration bound shrunk by RANSACUpdateNumIters(0.99, outlier ratio, 5, bound), and the final
// pose fitted on the best inlier set.  Each 5-point model and the final fit are the published EPnP (Lepetit, Moreno-Noguer
// and Fua, IJCV 2009) in fp64, with the control-point axes signed as OpenCV's SVD signs them (opencv_svd3); with 6 or
// more points that is cv2.solvePnP(EPNP)'s pose.  On 5 and 4 points the basis of MᵀM's exact null space is fixed here
// (null_space_basis), where OpenCV leaves it to rounding (INTEGRATION.md).
//
// One warp per person, one lane per hypothesis: hypotheses run in waves of 32, after each wave the lanes are scanned in
// iteration order with shuffles so that acceptance and the iteration bound follow the sequential loop exactly; most
// people stop after the first wave.  Each lane's 12x12 MᵀM and its Jacobi rotations live in shared memory.
#include "common.cuh"

namespace b200romp {
namespace {

constexpr int kJ = 24;            // SMPL joints used (utils.py:402 j3ds[:, :24])
constexpr int kModel = 5;         // EPnP's RANSAC model points (solvePnPRansac)
constexpr int kMaxIters = 100;    // iterationsCount (utils.py:341)
constexpr int kMinRansac = kModel + 1;
constexpr double kF = 443.4, kC = 256.0;
constexpr float kThresh2 = 400.f; // reprojectionError 20, squared (utils.py:341)
constexpr int kScratch = 288;     // per lane: 12x12 MᵀM + 12x12 eigenvectors

// The 100 subsets for every n in 6..24, drawn by OpenCV's RNG rule (state = (uint32)state * 4164903690 + (state >> 32),
// uniform(0, n) = next() % n, a repeat within a subset is drawn again) at compile time.
struct SubsetTable {
  unsigned char idx[kJ - kMinRansac + 1][kMaxIters][kModel];
};
constexpr SubsetTable make_subsets() {
  SubsetTable t{};
  for (int n = kMinRansac; n <= kJ; ++n) {
    unsigned long long s = ~0ull;
    for (int it = 0; it < kMaxIters; ++it)
      for (int i = 0; i < kModel;) {
        s = (unsigned long long)(unsigned)s * 4164903690ull + (s >> 32);
        const int v = (int)((unsigned)s % (unsigned)n);
        bool dup = false;
        for (int j = 0; j < i; ++j) dup = dup || t.idx[n - kMinRansac][it][j] == v;
        if (!dup) t.idx[n - kMinRansac][it][i++] = (unsigned char)v;
      }
  }
  return t;
}
constexpr SubsetTable kSubsetsHost = make_subsets();
__constant__ SubsetTable kSubsets = kSubsetsHost;

// the points of one person (compacted valid joints) in shared memory
struct Person {
  float pw[kJ][3];
  float p2[kJ][2];
};

// one lane's strided slice of the warp's scratch: element i at p[i * 32]
struct Lane {
  double* p;
  __device__ __forceinline__ double& operator[](int i) const { return p[i * 32]; }
};

// the pixel EPnP sees: cv2 undistorts to normalised coordinates of the input type (float32 for the RANSAC hypotheses,
// float64 for the final fit) and multiplies back by K
__device__ __forceinline__ double seen_pixel(float p, bool hypothesis) {
  double x = ((double)p - kC) * (1.0 / kF);
  if (hypothesis) x = (double)(float)x;
  return x * kF + kC;
}

// symmetric 3x3 eigen-decomposition by cyclic Jacobi; eigenvalues descending, v[k] = k-th eigenvector
__device__ __noinline__ void sym_eig3(double a[3][3], double w[3], double v[3][3]) {
  double V[3][3] = {{1, 0, 0}, {0, 1, 0}, {0, 0, 1}};
  for (int sweep = 0; sweep < 30; ++sweep) {
    const double off = a[0][1] * a[0][1] + a[0][2] * a[0][2] + a[1][2] * a[1][2];
    const double dia = a[0][0] * a[0][0] + a[1][1] * a[1][1] + a[2][2] * a[2][2];
    if (off <= 1e-34 * dia || off == 0.0) break;
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      const int p = r == 2 ? 1 : 0, q = r == 0 ? 1 : 2;
      const double apq = a[p][q];
      if (apq == 0.0) continue;
      const double th = (a[q][q] - a[p][p]) / (2.0 * apq);
      const double t = (th >= 0 ? 1.0 : -1.0) / (fabs(th) + sqrt(th * th + 1.0));
      const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        const double x = a[k][p], y = a[k][q];
        a[k][p] = c * x - s * y; a[k][q] = s * x + c * y;
      }
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        const double x = a[p][k], y = a[q][k];
        a[p][k] = c * x - s * y; a[q][k] = s * x + c * y;
      }
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        const double x = V[k][p], y = V[k][q];
        V[k][p] = c * x - s * y; V[k][q] = s * x + c * y;
      }
    }
  }
  int o[3] = {0, 1, 2};
  if (a[o[0]][o[0]] < a[o[1]][o[1]]) { const int t = o[0]; o[0] = o[1]; o[1] = t; }
  if (a[o[1]][o[1]] < a[o[2]][o[2]]) { const int t = o[1]; o[1] = o[2]; o[2] = t; }
  if (a[o[0]][o[0]] < a[o[1]][o[1]]) { const int t = o[0]; o[0] = o[1]; o[1] = t; }
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    w[k] = a[o[k]][o[k]];
#pragma unroll
    for (int j = 0; j < 3; ++j) v[k][j] = V[j][o[k]];
  }
}

// SVD of a symmetric 3x3 the way OpenCV's cvSVD computes it (one-sided Jacobi on the rows of Aᵀ, JacobiSVDImpl_ with
// eps = 10 DBL_EPSILON, then the rows sorted by norm and normalised).  EPnP's control points lie along these axes, and
// with noisy points the pose depends on the sign of each axis: this rule gives OpenCV's signs.  w descending, u[k] = row k.
__device__ __noinline__ void opencv_svd3(const double a[3][3], double w[3], double u[3][3]) {
  double At[3][3], W[3];
#pragma unroll
  for (int i = 0; i < 3; ++i) {
#pragma unroll
    for (int k = 0; k < 3; ++k) At[i][k] = a[k][i];
    W[i] = At[i][0] * At[i][0] + At[i][1] * At[i][1] + At[i][2] * At[i][2];
  }
  for (int iter = 0; iter < 30; ++iter) {
    bool changed = false;
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
      for (int j = i + 1; j < 3; ++j) {
        double p = At[i][0] * At[j][0] + At[i][1] * At[j][1] + At[i][2] * At[j][2];
        if (fabs(p) <= 10.0 * 2.220446049250313e-16 * sqrt(W[i] * W[j])) continue;
        p *= 2.0;
        const double beta = W[i] - W[j], gamma = hypot(p, beta);
        double c, s;
        if (beta < 0) {
          s = sqrt((gamma - beta) * 0.5 / gamma);
          c = p / (gamma * s * 2.0);
        } else {
          c = sqrt((gamma + beta) / (gamma * 2.0));
          s = p / (gamma * c * 2.0);
        }
        double na = 0.0, nb = 0.0;
#pragma unroll
        for (int k = 0; k < 3; ++k) {
          const double t0 = c * At[i][k] + s * At[j][k], t1 = -s * At[i][k] + c * At[j][k];
          At[i][k] = t0; At[j][k] = t1;
          na += t0 * t0; nb += t1 * t1;
        }
        W[i] = na; W[j] = nb;
        changed = true;
      }
    if (!changed) break;
  }
#pragma unroll
  for (int i = 0; i < 3; ++i) W[i] = sqrt(At[i][0] * At[i][0] + At[i][1] * At[i][1] + At[i][2] * At[i][2]);
  int o[3] = {0, 1, 2};
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    int j = i;
#pragma unroll
    for (int k = i + 1; k < 3; ++k)
      if (W[o[j]] < W[o[k]]) j = k;
    const int t = o[i]; o[i] = o[j]; o[j] = t;
  }
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    w[k] = W[o[k]];
    const double inv = W[o[k]] > 0.0 ? 1.0 / W[o[k]] : 0.0;
#pragma unroll
    for (int j = 0; j < 3; ++j) u[k][j] = At[o[k]][j] * inv;
  }
}

// least squares of a 6xK system by Householder QR (cv::solve DECOMP_SVD and epnp::qr_solve give the same minimiser)
template <int K>
__device__ __forceinline__ void lstsq6(double (&A)[6][K], double (&b)[6], double (&x)[K]) {
#pragma unroll
  for (int k = 0; k < K; ++k) {
    double nrm = 0.0;
#pragma unroll
    for (int i = k; i < 6; ++i) nrm += A[i][k] * A[i][k];
    nrm = sqrt(nrm);
    const double alpha = A[k][k] > 0 ? -nrm : nrm;
    double v[6];
#pragma unroll
    for (int i = 0; i < 6; ++i) v[i] = i < k ? 0.0 : (i == k ? A[k][k] - alpha : A[i][k]);
    double vv = 0.0;
#pragma unroll
    for (int i = k; i < 6; ++i) vv += v[i] * v[i];
    if (vv == 0.0) continue;
#pragma unroll
    for (int j = k; j < K; ++j) {
      double s = 0.0;
#pragma unroll
      for (int i = k; i < 6; ++i) s += v[i] * A[i][j];
      s = 2.0 * s / vv;
#pragma unroll
      for (int i = k; i < 6; ++i) A[i][j] -= s * v[i];
    }
    double s = 0.0;
#pragma unroll
    for (int i = k; i < 6; ++i) s += v[i] * b[i];
    s = 2.0 * s / vv;
#pragma unroll
    for (int i = k; i < 6; ++i) b[i] -= s * v[i];
  }
#pragma unroll
  for (int r = K - 1; r >= 0; --r) {
    double a = b[r];
#pragma unroll
    for (int k = r + 1; k < K; ++k) a -= A[r][k] * x[k];
    x[r] = a / A[r][r];
  }
}

// EPnP state shared by the three beta candidates of one solve
struct Epnp {
  const Person* P;
  unsigned mask;
  bool hyp;
  int n;
  double c0[3];       // centroid = control point 0 (and pw0 of estimate_R_and_t)
  double ci[3][3];    // inverse of [c1-c0 | c2-c0 | c3-c0]

  __device__ __forceinline__ void alphas(int i, double a[4]) const {
    const double d[3] = {P->pw[i][0] - c0[0], P->pw[i][1] - c0[1], P->pw[i][2] - c0[2]};
#pragma unroll
    for (int j = 0; j < 3; ++j) a[1 + j] = ci[j][0] * d[0] + ci[j][1] * d[1] + ci[j][2] * d[2];
    a[0] = 1.0 - a[1] - a[2] - a[3];
  }
};

// ccs from betas over the null vectors nv (S[0..47], nv_k[i] = S[12k+i]), then R, t and the mean reprojection error
__device__ __noinline__ double r_and_t(const Epnp& e, Lane S, const double B[4], double R[3][3], double t[3]) {
  double ccs[4][3];
#pragma unroll
  for (int j = 0; j < 4; ++j)
#pragma unroll
    for (int k = 0; k < 3; ++k) ccs[j][k] = B[0] * S[3 * j + k] + B[1] * S[12 + 3 * j + k] + B[2] * S[24 + 3 * j + k] + B[3] * S[36 + 3 * j + k];
  double a[4];
  e.alphas(__ffs(e.mask) - 1, a);
  if (a[0] * ccs[0][2] + a[1] * ccs[1][2] + a[2] * ccs[2][2] + a[3] * ccs[3][2] < 0.0) {   // solve_for_sign
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int k = 0; k < 3; ++k) ccs[j][k] = -ccs[j][k];
  }
  double pc0[3] = {0, 0, 0};
  for (unsigned m = e.mask; m; m &= m - 1) {
    e.alphas(__ffs(m) - 1, a);
#pragma unroll
    for (int k = 0; k < 3; ++k) pc0[k] += a[0] * ccs[0][k] + a[1] * ccs[1][k] + a[2] * ccs[2][k] + a[3] * ccs[3][k];
  }
#pragma unroll
  for (int k = 0; k < 3; ++k) pc0[k] /= e.n;
  double abt[3][3] = {{0, 0, 0}, {0, 0, 0}, {0, 0, 0}};
  for (unsigned m = e.mask; m; m &= m - 1) {
    const int i = __ffs(m) - 1;
    e.alphas(i, a);
    const double dw[3] = {e.P->pw[i][0] - e.c0[0], e.P->pw[i][1] - e.c0[1], e.P->pw[i][2] - e.c0[2]};
#pragma unroll
    for (int j = 0; j < 3; ++j) {
      const double dc = a[0] * ccs[0][j] + a[1] * ccs[1][j] + a[2] * ccs[2][j] + a[3] * ccs[3][j] - pc0[j];
#pragma unroll
      for (int k = 0; k < 3; ++k) abt[j][k] += dc * dw[k];
    }
  }
  // R = U Vᵀ of ABt = U Σ Vᵀ: V and Σ² from ABtᵀABt, U_k = ABt v_k / σ_k
  double ata[3][3], w[3], v[3][3], u[3][3];
#pragma unroll
  for (int r = 0; r < 3; ++r)
#pragma unroll
    for (int c = 0; c < 3; ++c) ata[r][c] = abt[0][r] * abt[0][c] + abt[1][r] * abt[1][c] + abt[2][r] * abt[2][c];
  sym_eig3(ata, w, v);
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const double sg = sqrt(fmax(w[k], 0.0));
    const double inv = sg > 0.0 ? 1.0 / sg : 0.0;
#pragma unroll
    for (int r = 0; r < 3; ++r) u[k][r] = (abt[r][0] * v[k][0] + abt[r][1] * v[k][1] + abt[r][2] * v[k][2]) * inv;
  }
  if (!(sqrt(fmax(w[2], 0.0)) > 1e-12 * sqrt(fmax(w[0], 0.0)))) {    // rank 2: complete U by the cross product
    u[2][0] = u[0][1] * u[1][2] - u[0][2] * u[1][1];
    u[2][1] = u[0][2] * u[1][0] - u[0][0] * u[1][2];
    u[2][2] = u[0][0] * u[1][1] - u[0][1] * u[1][0];
  }
#pragma unroll
  for (int r = 0; r < 3; ++r)
#pragma unroll
    for (int c = 0; c < 3; ++c) R[r][c] = u[0][r] * v[0][c] + u[1][r] * v[1][c] + u[2][r] * v[2][c];
  const double det = R[0][0] * R[1][1] * R[2][2] + R[0][1] * R[1][2] * R[2][0] + R[0][2] * R[1][0] * R[2][1] -
                     R[0][2] * R[1][1] * R[2][0] - R[0][1] * R[1][0] * R[2][2] - R[0][0] * R[1][2] * R[2][1];
  if (det < 0) { R[2][0] = -R[2][0]; R[2][1] = -R[2][1]; R[2][2] = -R[2][2]; }
#pragma unroll
  for (int r = 0; r < 3; ++r) t[r] = pc0[r] - (R[r][0] * e.c0[0] + R[r][1] * e.c0[1] + R[r][2] * e.c0[2]);
  double sum = 0.0;
  for (unsigned m = e.mask; m; m &= m - 1) {
    const int i = __ffs(m) - 1;
    const double X = e.P->pw[i][0], Y = e.P->pw[i][1], Z = e.P->pw[i][2];
    const double xc = R[0][0] * X + R[0][1] * Y + R[0][2] * Z + t[0];
    const double yc = R[1][0] * X + R[1][1] * Y + R[1][2] * Z + t[1];
    const double iz = 1.0 / (R[2][0] * X + R[2][1] * Y + R[2][2] * Z + t[2]);
    const double du = seen_pixel(e.P->p2[i][0], e.hyp) - (kC + kF * xc * iz);
    const double dv = seen_pixel(e.P->p2[i][1], e.hyp) - (kC + kF * yc * iz);
    sum += sqrt(du * du + dv * dv);
  }
  return sum / e.n;
}

// L (6x10) at S[48 + 10 r + c]
__device__ __noinline__ void gauss_newton(Lane S, const double rho[6], double B[4]) {
  for (int it = 0; it < 5; ++it) {
    double A[6][4], b[6], x[4];
#pragma unroll
    for (int i = 0; i < 6; ++i) {
      double r[10];
#pragma unroll
      for (int c = 0; c < 10; ++c) r[c] = S[48 + 10 * i + c];
      A[i][0] = 2 * r[0] * B[0] + r[1] * B[1] + r[3] * B[2] + r[6] * B[3];
      A[i][1] = r[1] * B[0] + 2 * r[2] * B[1] + r[4] * B[2] + r[7] * B[3];
      A[i][2] = r[3] * B[0] + r[4] * B[1] + 2 * r[5] * B[2] + r[8] * B[3];
      A[i][3] = r[6] * B[0] + r[7] * B[1] + r[8] * B[2] + 2 * r[9] * B[3];
      b[i] = rho[i] - (r[0] * B[0] * B[0] + r[1] * B[0] * B[1] + r[2] * B[1] * B[1] + r[3] * B[0] * B[2] + r[4] * B[1] * B[2] +
                       r[5] * B[2] * B[2] + r[6] * B[0] * B[3] + r[7] * B[1] * B[3] + r[8] * B[2] * B[3] + r[9] * B[3] * B[3]);
    }
    lstsq6<4>(A, b, x);
#pragma unroll
    for (int k = 0; k < 4; ++k) B[k] += x[k];
  }
}

// symmetric 4x4 eigen-decomposition by cyclic Jacobi; eigenvalues ascending, v[k] = k-th eigenvector
__device__ __noinline__ void sym_eig4(double a[4][4], double v[4][4]) {
  double V[4][4] = {{1, 0, 0, 0}, {0, 1, 0, 0}, {0, 0, 1, 0}, {0, 0, 0, 1}};
  for (int sweep = 0; sweep < 30; ++sweep) {
    bool rotated = false;
#pragma unroll
    for (int p = 0; p < 3; ++p)
#pragma unroll
      for (int q = p + 1; q < 4; ++q) {
        const double apq = a[p][q];
        if (fabs(apq) <= 1e-17 * sqrt(fabs(a[p][p] * a[q][q])) || apq == 0.0) continue;
        rotated = true;
        const double th = (a[q][q] - a[p][p]) / (2.0 * apq);
        const double t = (th >= 0 ? 1.0 : -1.0) / (fabs(th) + sqrt(th * th + 1.0));
        const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const double x = a[k][p], y = a[k][q];
          a[k][p] = c * x - s * y; a[k][q] = s * x + c * y;
        }
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const double x = a[p][k], y = a[q][k];
          a[p][k] = c * x - s * y; a[q][k] = s * x + c * y;
        }
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const double x = V[k][p], y = V[k][q];
          V[k][p] = c * x - s * y; V[k][q] = s * x + c * y;
        }
      }
    if (!rotated) break;
  }
  int o[4] = {0, 1, 2, 3};
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3 - i; ++j)
      if (a[o[j + 1]][o[j + 1]] < a[o[j]][o[j]]) { const int t = o[j]; o[j] = o[j + 1]; o[j + 1] = t; }
#pragma unroll
  for (int k = 0; k < 4; ++k)
#pragma unroll
    for (int j = 0; j < 4; ++j) v[k][j] = V[j][o[k]];
}

// With fewer than 6 points MᵀM has an exact null space of d = 12 - 2n dimensions (5 points: 2, 4 points: 4), whose basis
// the published method leaves to the eigen-solver, and EPnP's beta approximations depend on that basis.  It is fixed here
// as the eigenvectors, ascending, of diag(1..12) restricted to the null space, so that the pose does not depend on how
// the solver happened to rotate within it (the restatement in tests/pnp_oracle.py does the same).
__device__ void null_space_basis(Lane S, int d) {
  double b[4][4], E[4][4];
#pragma unroll
  for (int x = 0; x < 4; ++x)
#pragma unroll
    for (int y = 0; y < 4; ++y) {
      double acc = 0.0;
      if (x < d && y < d)
        for (int i = 0; i < 12; ++i) acc += (i + 1) * S[12 * x + i] * S[12 * y + i];
      else if (x == y)
        acc = 1e300 * (x + 1);            // outside the null space: stays in place, sorted last
      b[x][y] = acc;
    }
  sym_eig4(b, E);
  for (int i = 0; i < 12; ++i) {
    double r[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) r[k] = E[k][0] * S[i] + E[k][1] * S[12 + i] + E[k][2] * S[24 + i] + E[k][3] * S[36 + i];
#pragma unroll
    for (int k = 0; k < 4; ++k) S[12 * k + i] = r[k];
  }
}

// EPnP on the points of ``mask`` (bit i = compacted joint i); S: this lane's 288-double scratch.  Returns R, t.
__device__ void epnp(const Person* P, unsigned mask, bool hyp, Lane S, double R[3][3], double t[3]) {
  Epnp e;
  e.P = P; e.mask = mask; e.hyp = hyp; e.n = __popc(mask);
  // choose_control_points: centroid + principal axes scaled by sqrt(eigenvalue / n)
  double c0[3] = {0, 0, 0};
  for (unsigned m = mask; m; m &= m - 1) {
    const int i = __ffs(m) - 1;
#pragma unroll
    for (int k = 0; k < 3; ++k) c0[k] += P->pw[i][k];
  }
#pragma unroll
  for (int k = 0; k < 3; ++k) e.c0[k] = c0[k] / e.n;
  double cov[3][3] = {{0, 0, 0}, {0, 0, 0}, {0, 0, 0}};
  for (unsigned m = mask; m; m &= m - 1) {
    const int i = __ffs(m) - 1;
    const double d[3] = {P->pw[i][0] - e.c0[0], P->pw[i][1] - e.c0[1], P->pw[i][2] - e.c0[2]};
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
      for (int c = 0; c < 3; ++c) cov[r][c] += d[r] * d[c];
  }
  double dc[3], uc[3][3], cws[4][3];
  opencv_svd3(cov, dc, uc);
#pragma unroll
  for (int k = 0; k < 3; ++k) cws[0][k] = e.c0[k];
#pragma unroll
  for (int i = 1; i < 4; ++i) {
    const double s = sqrt(fmax(dc[i - 1], 0.0) / e.n);
#pragma unroll
    for (int k = 0; k < 3; ++k) cws[i][k] = e.c0[k] + s * uc[i - 1][k];
  }
  // compute_barycentric_coordinates: CC[r][c] = cws[c+1][r] - cws[0][r], ci = CC⁻¹
  {
    double cc[3][3];
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
      for (int c = 0; c < 3; ++c) cc[r][c] = cws[c + 1][r] - cws[0][r];
    const double det = cc[0][0] * (cc[1][1] * cc[2][2] - cc[1][2] * cc[2][1]) - cc[0][1] * (cc[1][0] * cc[2][2] - cc[1][2] * cc[2][0]) +
                       cc[0][2] * (cc[1][0] * cc[2][1] - cc[1][1] * cc[2][0]);
    const double id = 1.0 / det;
    e.ci[0][0] = (cc[1][1] * cc[2][2] - cc[1][2] * cc[2][1]) * id;
    e.ci[0][1] = (cc[0][2] * cc[2][1] - cc[0][1] * cc[2][2]) * id;
    e.ci[0][2] = (cc[0][1] * cc[1][2] - cc[0][2] * cc[1][1]) * id;
    e.ci[1][0] = (cc[1][2] * cc[2][0] - cc[1][0] * cc[2][2]) * id;
    e.ci[1][1] = (cc[0][0] * cc[2][2] - cc[0][2] * cc[2][0]) * id;
    e.ci[1][2] = (cc[0][2] * cc[1][0] - cc[0][0] * cc[1][2]) * id;
    e.ci[2][0] = (cc[1][0] * cc[2][1] - cc[1][1] * cc[2][0]) * id;
    e.ci[2][1] = (cc[0][1] * cc[2][0] - cc[0][0] * cc[2][1]) * id;
    e.ci[2][2] = (cc[0][0] * cc[1][1] - cc[0][1] * cc[1][0]) * id;
  }
  // MᵀM (upper triangle, mirrored below) into S[0..143]; V = I into S[144..287]
  for (int i = 0; i < 144; ++i) { S[i] = 0.0; S[144 + i] = (i % 13 == 0) ? 1.0 : 0.0; }
  for (unsigned m = mask; m; m &= m - 1) {
    const int i = __ffs(m) - 1;
    double a[4];
    e.alphas(i, a);
    const double du = kC - seen_pixel(P->p2[i][0], hyp), dv = kC - seen_pixel(P->p2[i][1], hyp);
    double r1[12], r2[12];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      r1[3 * j] = a[j] * kF; r1[3 * j + 1] = 0.0; r1[3 * j + 2] = a[j] * du;
      r2[3 * j] = 0.0; r2[3 * j + 1] = a[j] * kF; r2[3 * j + 2] = a[j] * dv;
    }
#pragma unroll
    for (int r = 0; r < 12; ++r)
#pragma unroll
      for (int c = r; c < 12; ++c) S[r * 12 + c] += r1[r] * r1[c] + r2[r] * r2[c];
  }
  for (int r = 1; r < 12; ++r)
    for (int c = 0; c < r; ++c) S[r * 12 + c] = S[c * 12 + r];
  // cyclic Jacobi on MᵀM; a rotation is skipped when the pair is already decoupled to working precision
  double scale = 0.0;
  for (int k = 0; k < 12; ++k) scale = fmax(scale, fabs(S[k * 13]));
  for (int sweep = 0; sweep < 30; ++sweep) {
    bool rotated = false;
    for (int p = 0; p < 11; ++p)
      for (int q = p + 1; q < 12; ++q) {
        const double apq = S[p * 12 + q], app = S[p * 13], aqq = S[q * 13];
        if (fabs(apq) <= 1e-17 * sqrt(fabs(app * aqq)) || fabs(apq) <= 1e-300 + 1e-30 * scale) continue;
        rotated = true;
        const double th = (aqq - app) / (2.0 * apq);
        const double tt = (th >= 0 ? 1.0 : -1.0) / (fabs(th) + sqrt(th * th + 1.0));
        const double c = 1.0 / sqrt(tt * tt + 1.0), s = tt * c;
        for (int k = 0; k < 12; ++k) {
          const double x = S[k * 12 + p], y = S[k * 12 + q];
          S[k * 12 + p] = c * x - s * y; S[k * 12 + q] = s * x + c * y;
        }
        for (int k = 0; k < 12; ++k) {
          const double x = S[p * 12 + k], y = S[q * 12 + k];
          S[p * 12 + k] = c * x - s * y; S[q * 12 + k] = s * x + c * y;
        }
        for (int k = 0; k < 12; ++k) {
          const double x = S[144 + k * 12 + p], y = S[144 + k * 12 + q];
          S[144 + k * 12 + p] = c * x - s * y; S[144 + k * 12 + q] = s * x + c * y;
        }
      }
    if (!rotated) break;
  }
  // the 4 smallest eigenvalues, ascending: nv_0 (smallest) .. nv_3 -> S[12k + i]
  int o[4];
  {
    unsigned used = 0;
    for (int k = 0; k < 4; ++k) {
      int best = -1;
      for (int j = 0; j < 12; ++j)
        if (!(used >> j & 1) && (best < 0 || S[j * 13] < S[best * 13])) best = j;
      used |= 1u << best;
      o[k] = best;
    }
  }
  for (int k = 0; k < 4; ++k)
    for (int i = 0; i < 12; ++i) S[12 * k + i] = S[144 + i * 12 + o[k]];
  if (e.n < 6) null_space_basis(S, 12 - 2 * e.n);
  // compute_L_6x10 (into S[48..107]) / compute_rho over the control-point pairs (0,1) (0,2) (0,3) (1,2) (1,3) (2,3)
  double rho[6];
  {
    const int pa[6] = {0, 0, 0, 1, 1, 2}, pb[6] = {1, 2, 3, 2, 3, 3};
#pragma unroll
    for (int r = 0; r < 6; ++r) {
      double dv[4][3];
#pragma unroll
      for (int k = 0; k < 4; ++k)
#pragma unroll
        for (int c = 0; c < 3; ++c) dv[k][c] = S[12 * k + 3 * pa[r] + c] - S[12 * k + 3 * pb[r] + c];
      auto dot = [&](int x, int y) { return dv[x][0] * dv[y][0] + dv[x][1] * dv[y][1] + dv[x][2] * dv[y][2]; };
      const double l[10] = {dot(0, 0), 2 * dot(0, 1), dot(1, 1), 2 * dot(0, 2), 2 * dot(1, 2),
                            dot(2, 2), 2 * dot(0, 3), 2 * dot(1, 3), 2 * dot(2, 3), dot(3, 3)};
#pragma unroll
      for (int c = 0; c < 10; ++c) S[48 + 10 * r + c] = l[c];
      double d2 = 0.0;
#pragma unroll
      for (int c = 0; c < 3; ++c) d2 += (cws[pa[r]][c] - cws[pb[r]][c]) * (cws[pa[r]][c] - cws[pb[r]][c]);
      rho[r] = d2;
    }
  }
  double best_err = 0.0;
#pragma unroll 1
  for (int cand = 0; cand < 3; ++cand) {
    double B[4] = {0, 0, 0, 0};
    if (cand == 0) {                      // find_betas_approx_1: [B11 B12 B13 B14]
      double A[6][4], b[6], x[4];
#pragma unroll
      for (int i = 0; i < 6; ++i) { A[i][0] = S[48 + 10 * i]; A[i][1] = S[49 + 10 * i]; A[i][2] = S[51 + 10 * i]; A[i][3] = S[54 + 10 * i]; b[i] = rho[i]; }
      lstsq6<4>(A, b, x);
      const double b0 = sqrt(fabs(x[0])), sg = x[0] < 0 ? -1.0 : 1.0;
      B[0] = b0; B[1] = sg * x[1] / b0; B[2] = sg * x[2] / b0; B[3] = sg * x[3] / b0;
    } else if (cand == 1) {               // find_betas_approx_2: [B11 B12 B22]
      double A[6][3], b[6], x[3];
#pragma unroll
      for (int i = 0; i < 6; ++i) { A[i][0] = S[48 + 10 * i]; A[i][1] = S[49 + 10 * i]; A[i][2] = S[50 + 10 * i]; b[i] = rho[i]; }
      lstsq6<3>(A, b, x);
      if (x[0] < 0) { B[0] = sqrt(-x[0]); B[1] = x[2] < 0 ? sqrt(-x[2]) : 0.0; }
      else { B[0] = sqrt(x[0]); B[1] = x[2] > 0 ? sqrt(x[2]) : 0.0; }
      if (x[1] < 0) B[0] = -B[0];
    } else {                              // find_betas_approx_3: [B11 B12 B22 B13 B23]
      double A[6][5], b[6], x[5];
#pragma unroll
      for (int i = 0; i < 6; ++i) { for (int k = 0; k < 5; ++k) A[i][k] = S[48 + 10 * i + k]; b[i] = rho[i]; }
      lstsq6<5>(A, b, x);
      if (x[0] < 0) { B[0] = sqrt(-x[0]); B[1] = x[2] < 0 ? sqrt(-x[2]) : 0.0; }
      else { B[0] = sqrt(x[0]); B[1] = x[2] > 0 ? sqrt(x[2]) : 0.0; }
      if (x[1] < 0) B[0] = -B[0];
      B[2] = x[3] / B[0];
    }
    gauss_newton(S, rho, B);
    double Rc[3][3], tc[3];
    const double err = r_and_t(e, S, B, Rc, tc);
    if (cand == 0 || err < best_err) {
      best_err = err;
#pragma unroll
      for (int r = 0; r < 3; ++r) {
        t[r] = tc[r];
#pragma unroll
        for (int c = 0; c < 3; ++c) R[r][c] = Rc[r][c];
      }
    }
  }
}

// findInliers: the projection in double rounded to float32, dx*dx + dy*dy in float32 without contraction, <= 400
__device__ unsigned inliers(const Person* P, int n, const double R[3][3], const double t[3]) {
  unsigned m = 0;
  for (int i = 0; i < n; ++i) {
    const double X = P->pw[i][0], Y = P->pw[i][1], Z = P->pw[i][2];
    const double iz = 1.0 / (R[2][0] * X + R[2][1] * Y + R[2][2] * Z + t[2]);
    const float u = (float)((R[0][0] * X + R[0][1] * Y + R[0][2] * Z + t[0]) * iz * kF + kC);
    const float v = (float)((R[1][0] * X + R[1][1] * Y + R[1][2] * Z + t[1]) * iz * kF + kC);
    const float dx = __fsub_rn(P->p2[i][0], u), dy = __fsub_rn(P->p2[i][1], v);
    if (__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)) <= kThresh2) m |= 1u << i;
  }
  return m;
}

// cv::RANSACUpdateNumIters
__device__ int update_num_iters(double p, double ep, int model_points, int max_iters) {
  const double num = log(fmax(1.0 - p, 2.2250738585072014e-308));
  double denom = 1.0 - pow(1.0 - ep, (double)model_points);
  if (denom < 2.2250738585072014e-308) return 0;
  denom = log(denom);
  return denom >= 0 || -num >= max_iters * (-denom) ? max_iters : __double2int_rn(num / denom);
}

__global__ void __launch_bounds__(32) cam_trans_pnp_kernel(const float* __restrict__ joints, const float* __restrict__ cam, int n_host,
                                                           const int* __restrict__ d_count, float* __restrict__ out,
                                                           int* __restrict__ out_mask) {
  extern __shared__ double scratch[];
  __shared__ Person P;
  const int person = blockIdx.x, lane = threadIdx.x;
  const int N = d_count ? min(n_host, *d_count) : n_host;
  if (person >= N) return;
  // valid joints (utils.py:404-419): pj2d = (xy * s + t + 1) * 256 in fp32 (post_parser.py:98), pj2d_y > -2 and z != -2
  const float s = cam[person * 3 + 0], tx = cam[person * 3 + 1], ty = cam[person * 3 + 2];
  bool valid = false;
  float x = 0.f, y = 0.f, z = 0.f, px = 0.f, py = 0.f;
  if (lane < kJ) {
    const float* q = joints + ((size_t)person * 71 + lane) * 3;
    x = q[0]; y = q[1]; z = q[2];
    px = __fmul_rn(__fadd_rn(__fadd_rn(__fmul_rn(x, s), tx), 1.f), 256.f);
    py = __fmul_rn(__fadd_rn(__fadd_rn(__fmul_rn(y, s), ty), 1.f), 256.f);
    valid = py > -2.f && z != -2.f;
  }
  const unsigned vb = __ballot_sync(0xffffffffu, valid);
  const int n = __popc(vb);
  if (valid) {
    const int k = __popc(vb & ((1u << lane) - 1u));
    P.pw[k][0] = x; P.pw[k][1] = y; P.pw[k][2] = z;
    P.p2[k][0] = px; P.p2[k][1] = py;
  }
  __syncwarp();
  float* o = out + (size_t)person * 3;
  if (n < 4) {                                          // utils.py:420-422
    if (lane == 0) {
      o[0] = o[1] = o[2] = -1.f;
      if (out_mask) out_mask[person] = 0;
    }
    return;
  }
  const Lane S{scratch + lane};
  const unsigned all = n == 32 ? 0xffffffffu : (1u << n) - 1u;
  unsigned best_mask = 0;
  bool hyp_final = false;
  if (n <= kModel) {                                    // solvePnPRansac: the kernel on every point, all inliers
    best_mask = all;
    hyp_final = true;
  } else {
    int best = 0, niters = kMaxIters;
    for (int wave = 0; wave * 32 < niters; ++wave) {
      const int it = wave * 32 + lane;
      int good = 0;
      unsigned m = 0;
      if (it < niters) {
        const unsigned char* sub = kSubsets.idx[n - kMinRansac][it];
        unsigned sm = 0;
#pragma unroll
        for (int k = 0; k < kModel; ++k) sm |= 1u << sub[k];
        double R[3][3], t[3];
        epnp(&P, sm, true, S, R, t);
        m = inliers(&P, n, R, t);
        good = __popc(m);
      }
      // the sequential acceptance rule over this wave's iterations, in order
      for (int l = 0; l < 32; ++l) {
        const int g = __shfl_sync(0xffffffffu, good, l);
        const unsigned gm = __shfl_sync(0xffffffffu, m, l);
        if (wave * 32 + l >= niters) break;
        if (g > max(best, kModel - 1)) {
          best = g;
          best_mask = gm;
          niters = update_num_iters(0.99, (double)(n - g) / n, kModel, niters);
        }
      }
    }
  }
  if (lane == 0) {
    if (best_mask == 0) {                               // no model accepted: inliers is None (utils.py:342-343)
      o[0] = o[1] = o[2] = -1.f;
    } else {
      double R[3][3], t[3];
      epnp(&P, best_mask, hyp_final, S, R, t);
      o[0] = (float)t[0]; o[1] = (float)t[1]; o[2] = (float)t[2];
    }
    if (out_mask) out_mask[person] = (int)best_mask;
  }
}

}  // namespace
}  // namespace b200romp

using namespace b200romp;

extern "C" int b200romp_cam_trans_pnp(const float* joints, const float* cam, int n, const int* d_count, float* cam_trans,
                                      int* inlier_mask, b200romp_stream stream) {
  B2R_REQUIRE(joints && cam && cam_trans && n > 0, "cam_trans_pnp: bad arguments");
  const size_t smem = (size_t)kScratch * 32 * sizeof(double);
  B2R_CUDA_OK(cudaFuncSetAttribute(cam_trans_pnp_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  cam_trans_pnp_kernel<<<n, 32, smem, (cudaStream_t)stream>>>(joints, cam, n, d_count, cam_trans, inlier_mask);
  B2R_CUDA_OK(cudaGetLastError());
  return B200ROMP_OK;
}
