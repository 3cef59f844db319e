// Absolute camera pose from 2D-3D matches on the device: P3P RANSAC with Gauss-Newton local optimisation for a batch
// of queries, and the lift of a database cutout's matched pixels to 3D through its scan (hloc's InLoc pipeline,
// pose_from_cluster / interpolate_scan).
//
// p2p_find_absolute_pose_batch enqueues, with the query as grid dimension y:
//   abs_prep_kernel   (1 block)          effective row count, finiteness, the centroid of the world points, fp32 rows
//                                        (world points minus the centroid, pixels minus the principal point)
//   abs_round_kernel  (cdiv(count, 8))   per round: 3-row samples -> Grunert's P3P quartic (up to 4 poses, one thread
//                                        per sample), every (pose, row) scored in fp32
//   abs_select_kernel (1 block)          ransac_common.cuh's select_round on 12-double poses, the stopping bound (s = 3)
//   abs_lo_kernel     (1 block)          Gauss-Newton on the inliers of the winner, kept while the count grows; outputs
// The solver and scorer are their own (rows of 5 values, models of 12), so the two-view kinds of verify_common.cuh do
// not branch on this caller.  Everything a query computes depends on its rows, threshold and cameras alone, every
// combine runs in a fixed order and no grid size depends on the device: results are bit-reproducible, and a query's
// result is the same alone or in a batch.  Restated in oracle/abspose_oracle.py.
#include <algorithm>

#include <math.h>

#include "kernels.h"
#include "ransac_common.cuh"

namespace p2p {
namespace {

constexpr int kAbsRound = 1024;      // hypotheses per round
constexpr int kAbsSample = 3;        // rows per minimal sample
constexpr int kAbsSlots = 4;         // P3P poses per sample
constexpr int kAbsMinRows = 4;       // fewer rows: no rounds, no model
constexpr int kAbsHypPerBlock = 8;   // samples solved (one thread each) and scored per block
constexpr int kAbsThreads = 256;     // 8 warps
constexpr int kAbsTile = 1024;       // fp32 rows staged in shared memory per scoring pass
constexpr int kAbsLoIters = 4;       // local-optimisation refits
constexpr int kAbsGnSteps = 3;       // Gauss-Newton steps per refit
constexpr int kAbsLoThreads = 256;
constexpr int kLiftThreads = 1024;
constexpr size_t kAbsModels = (size_t)kAbsRound * kAbsSlots * 12;   // doubles of round models per query
constexpr size_t kAbsCounts = (size_t)kAbsRound * kAbsSlots;        // ints of round counts per query

struct __align__(8) AbsRow32 {       // scoring row: world point minus the centroid, pixel minus the principal point
  float X, Y, Z, du, dv, pad;
};

struct AbsState {
  double best[12];                   // best pose so far in the centred frame: R row-major, then t (x = R (X - c) + t)
  double mean[3];                    // centroid c of the world points
  double fx, fy, cx, cy;             // the query's camera
  int n;                             // effective row count
  int bad;                           // a value is not finite
  int stop;                          // no further rounds are needed
  int best_count;                    // 0: no model yet
  int n_all;                         // rows of the query (mask length)
  long long row0;                    // first row of the query in the row array and the mask
  long long row32;                   // first row of the query in rows32
  float th2;                         // squared pixel threshold
};

// ---- P3P: Grunert's quartic as given in Haralick et al., "Review and analysis of solutions of the three point
// perspective pose estimation problem" (IJCV 1994), one thread, fp64 -------------------------------------------------

// Largest real root of m^3 + b m^2 + c m + d (trigonometric form for three real roots, Cardano for one).
__device__ double cubic_max_root(double b, double c, double d) {
  const double p = c - b * b / 3.0, q = 2.0 * b * b * b / 27.0 - b * c / 3.0 + d, shift = -b / 3.0;
  const double disc = q * q / 4.0 + p * p * p / 27.0;
  if (disc > 0.0) {
    const double sq = sqrt(disc);
    return cbrt(-q / 2.0 + sq) + cbrt(-q / 2.0 - sq) + shift;
  }
  if (p >= 0.0) return shift;
  const double rr = 2.0 * sqrt(-p / 3.0);
  const double phi = acos(fmin(1.0, fmax(-1.0, 1.5 * q / p * sqrt(-3.0 / p)))) / 3.0;
  return rr * cos(phi) + shift;
}

// Real roots of A4 v^4 + A3 v^3 + A2 v^2 + A1 v + A0 by Ferrari's method (the resolvent's largest root), each polished
// by two Newton steps, ascending.  0 roots when the leading coefficient vanishes against the others.
__device__ int quartic_roots(const double (&A)[5], double (&r)[4]) {
  const double amax = fmax(fmax(fabs(A[0]), fabs(A[1])), fmax(fmax(fabs(A[2]), fabs(A[3])), fabs(A[4])));
  if (!(fabs(A[4]) > 1e-12 * amax)) return 0;
  const double b = A[3] / A[4], c = A[2] / A[4], d = A[1] / A[4], e = A[0] / A[4];
  const double p = c - 3.0 * b * b / 8.0, q = b * b * b / 8.0 - b * c / 2.0 + d;
  const double rr = -3.0 * b * b * b * b / 256.0 + b * b * c / 16.0 - b * d / 4.0 + e;
  const double m = cubic_max_root(p, p * p / 4.0 - rr, -q * q / 8.0);
  if (!(m > 0.0)) return 0;
  const double s = sqrt(2.0 * m);
  int nr = 0;
  for (int k = 0; k < 2; ++k) {
    const double sg = k == 0 ? 1.0 : -1.0;
    const double B = -sg * s, C = p / 2.0 + m + sg * q / (2.0 * s);
    const double D = B * B - 4.0 * C;
    if (!(D >= 0.0)) continue;
    const double sd = sqrt(D);
    r[nr++] = (-B + sd) / 2.0 - b / 4.0;
    r[nr++] = (-B - sd) / 2.0 - b / 4.0;
  }
  for (int k = 0; k < nr; ++k)
    for (int it = 0; it < 2; ++it) {
      const double v = r[k];
      const double f = (((A[4] * v + A[3]) * v + A[2]) * v + A[1]) * v + A[0];
      const double df = ((4.0 * A[4] * v + 3.0 * A[3]) * v + 2.0 * A[2]) * v + A[1];
      if (df != 0.0) r[k] = v - f / df;
    }
  for (int i = 1; i < nr; ++i)
    for (int k = i; k > 0 && r[k] < r[k - 1]; --k) { const double t = r[k]; r[k] = r[k - 1]; r[k - 1] = t; }
  return nr;
}

__device__ __forceinline__ void sub3(const double* a, const double* b, double* c) {
  for (int i = 0; i < 3; ++i) c[i] = a[i] - b[i];
}
__device__ __forceinline__ void cross3d(const double* a, const double* b, double* c) {
  c[0] = a[1] * b[2] - a[2] * b[1];
  c[1] = a[2] * b[0] - a[0] * b[2];
  c[2] = a[0] * b[1] - a[1] * b[0];
}
__device__ __forceinline__ double norm3(const double* a) { return sqrt(a[0] * a[0] + a[1] * a[1] + a[2] * a[2]); }

// Orthonormal frame of a triangle, columns e1 = (Q1 - Q0) / |.|, e2 = e3 x e1, e3 = (Q1 - Q0) x (Q2 - Q0) / |.|, as
// F[i][j] = e_j[i].  False for a degenerate triangle.
__device__ bool tri_frame(const double (&Q)[3][3], double (&F)[3][3]) {
  double e1[3], d2[3], e3[3], e2[3];
  sub3(Q[1], Q[0], e1);
  sub3(Q[2], Q[0], d2);
  cross3d(e1, d2, e3);
  const double n1 = norm3(e1), n3 = norm3(e3);
  if (!(n1 > 0.0) || !(n3 > 0.0)) return false;
  for (int i = 0; i < 3; ++i) { e1[i] /= n1; e3[i] /= n3; }
  cross3d(e3, e1, e2);
  for (int i = 0; i < 3; ++i) { F[i][0] = e1[i]; F[i][1] = e2[i]; F[i][2] = e3[i]; }
  return true;
}

// Bearings j[3] (unit vectors) and world points X[3] (centred) -> up to 4 poses (R row-major, t: s_i j_i = R X_i + t),
// in ascending order of the quartic's root v = s3 / s1.  A root is kept when u = s2 / s1, v and s1^2 are positive and
// the pose is finite.
__device__ int solve_p3p(const double (&j)[3][3], const double (&X)[3][3], double (&out)[kAbsSlots][12]) {
  double d[3];
  sub3(X[1], X[2], d);
  const double a2 = d[0] * d[0] + d[1] * d[1] + d[2] * d[2];
  sub3(X[0], X[2], d);
  const double b2 = d[0] * d[0] + d[1] * d[1] + d[2] * d[2];
  sub3(X[0], X[1], d);
  const double c2 = d[0] * d[0] + d[1] * d[1] + d[2] * d[2];
  if (!(b2 > 0.0)) return 0;
  const double ca = j[1][0] * j[2][0] + j[1][1] * j[2][1] + j[1][2] * j[2][2];
  const double cb = j[0][0] * j[2][0] + j[0][1] * j[2][1] + j[0][2] * j[2][2];
  const double cg = j[0][0] * j[1][0] + j[0][1] * j[1][1] + j[0][2] * j[1][2];
  const double amc = (a2 - c2) / b2, apc = (a2 + c2) / b2, bmc = (b2 - c2) / b2, bma = (b2 - a2) / b2;
  const double c2b = c2 / b2, a2b = a2 / b2;
  double A[5];
  A[4] = (amc - 1.0) * (amc - 1.0) - 4.0 * c2b * ca * ca;
  A[3] = 4.0 * (amc * (1.0 - amc) * cb - (1.0 - apc) * ca * cg + 2.0 * c2b * ca * ca * cb);
  A[2] = 2.0 * (amc * amc - 1.0 + 2.0 * amc * amc * cb * cb + 2.0 * bmc * ca * ca - 4.0 * apc * ca * cb * cg +
                2.0 * bma * cg * cg);
  A[1] = 4.0 * (-amc * (1.0 + amc) * cb + 2.0 * a2b * cg * cg * cb - (1.0 - apc) * ca * cg);
  A[0] = (1.0 + amc) * (1.0 + amc) - 4.0 * a2b * cg * cg;
  double r[4];
  const int nr = quartic_roots(A, r);
  double FX[3][3];
  if (!tri_frame(X, FX)) return 0;
  int ns = 0;
  for (int k = 0; k < nr; ++k) {
    const double v = r[k];
    const double u = ((-1.0 + amc) * v * v - 2.0 * amc * cb * v + 1.0 + amc) / (2.0 * (cg - v * ca));
    const double s1sq = b2 / (1.0 + v * v - 2.0 * v * cb);
    if (!(u > 0.0 && v > 0.0 && s1sq > 0.0)) continue;
    const double s1 = sqrt(s1sq), s[3] = {s1, u * s1, v * s1};
    double P[3][3], FP[3][3];
    for (int i = 0; i < 3; ++i)
      for (int c = 0; c < 3; ++c) P[i][c] = s[i] * j[i][c];
    if (!tri_frame(P, FP)) continue;
    double* o = out[ns];
    bool ok = true;
    for (int a = 0; a < 3; ++a)
      for (int b = 0; b < 3; ++b) {      // R = FP FX^T
        o[3 * a + b] = FP[a][0] * FX[b][0] + FP[a][1] * FX[b][1] + FP[a][2] * FX[b][2];
        ok &= isfinite(o[3 * a + b]);
      }
    for (int a = 0; a < 3; ++a) {        // t = P0 - R X0
      o[9 + a] = P[0][a] - (o[3 * a] * X[0][0] + o[3 * a + 1] * X[0][1] + o[3 * a + 2] * X[0][2]);
      ok &= isfinite(o[9 + a]);
    }
    if (ok) ++ns;
  }
  return ns;
}

// ---- scoring ------------------------------------------------------------------------------------------------------
// fp32 projection of a pose: rows fx (R_0, t_0), fy (R_1, t_1), (R_2, t_2).
__device__ __forceinline__ void abs_proj32(const AbsState& S, const double* m, float* p) {
  for (int k = 0; k < 4; ++k) {
    p[k] = (float)(S.fx * (k < 3 ? m[k] : m[9]));
    p[4 + k] = (float)(S.fy * (k < 3 ? m[3 + k] : m[10]));
    p[8 + k] = (float)(k < 3 ? m[6 + k] : m[11]);
  }
}

// Depth z > 0 and squared reprojection error < th^2, as (a - du z)^2 + (b - dv z)^2 < th^2 z^2.
__device__ __forceinline__ bool abs_inlier(const float* p, const AbsRow32& r, float th2) {
  const float a = p[0] * r.X + p[1] * r.Y + p[2] * r.Z + p[3];
  const float b = p[4] * r.X + p[5] * r.Y + p[6] * r.Z + p[7];
  const float z = p[8] * r.X + p[9] * r.Y + p[10] * r.Z + p[11];
  const float eu = a - r.du * z, ev = b - r.dv * z;
  return z > 0.f && eu * eu + ev * ev < th2 * z * z;
}

// Bearing of row p (unit vector of ((u - cx) / fx, (v - cy) / fy, 1)) and its centred world point.
__device__ __forceinline__ void abs_row64(const AbsState& S, const double* p, double* j, double* X) {
  const double x = (p[0] - S.cx) / S.fx, y = (p[1] - S.cy) / S.fy;
  const double nj = sqrt(x * x + y * y + 1.0);
  j[0] = x / nj;
  j[1] = y / nj;
  j[2] = 1.0 / nj;
  for (int i = 0; i < 3; ++i) X[i] = p[2 + i] - S.mean[i];
}

// ---- kernels ------------------------------------------------------------------------------------------------------
struct Cam4 {
  double fx, fy, cx, cy;
};

// Query q: its camera intr[4 q ..] (fx, fy, cx, cy; device), or K1 when intr is null, and its threshold px_th_dev[q]
// (device), or px_th when px_th_dev is null.
__global__ void __launch_bounds__(1024) abs_prep_kernel(PairBatch B, const double* __restrict__ intr, Cam4 K1,
                                                        double px_th, const double* __restrict__ px_th_dev,
                                                        AbsRow32* __restrict__ rows32_all, AbsState* __restrict__ st_all) {
  __shared__ double red[33];
  __shared__ int s_n;
  const int tid = threadIdx.x, q = blockIdx.y;
  AbsState* st = st_all + q;
  const PairRange pr = pair_range(B, q);
  const int n = pr.n, stride = B.stride;
  const double* rows = B.rows + pr.row0 * stride;
  AbsRow32* rows32 = rows32_all + (pr.row0 - B.base);
  if (tid == 0) s_n = effective_rows(B, q, n);
  __syncthreads();
  const int m = s_n;
  double sx[3] = {0.0, 0.0, 0.0};
  int bad = 0;
  for (int r = tid; r < m; r += 1024) {
    const double* p = rows + (size_t)r * stride;
    bool fin = true;
    for (int k = 0; k < 5; ++k) fin &= isfinite(p[k]);
    bad |= !fin;
    for (int k = 0; k < 3; ++k) sx[k] += p[2 + k];
  }
  bad = __syncthreads_or(bad);
  double mean[3];
  for (int k = 0; k < 3; ++k) mean[k] = block_sum_1024(sx[k], red) / (double)(m > 0 ? m : 1);
  const double* k4 = intr + 4 * (size_t)q;
  const double fx = intr ? k4[0] : K1.fx, fy = intr ? k4[1] : K1.fy, cx = intr ? k4[2] : K1.cx,
               cy = intr ? k4[3] : K1.cy;
  for (int r = tid; r < m; r += 1024) {
    const double* p = rows + (size_t)r * stride;
    rows32[r] = AbsRow32{(float)(p[2] - mean[0]), (float)(p[3] - mean[1]), (float)(p[4] - mean[2]), (float)(p[0] - cx),
                         (float)(p[1] - cy), 0.f};
  }
  if (tid == 0) {
    if (px_th_dev != nullptr) px_th = px_th_dev[q];
    for (int j = 0; j < 12; ++j) st->best[j] = 0.0;
    for (int k = 0; k < 3; ++k) st->mean[k] = mean[k];
    st->fx = fx;
    st->fy = fy;
    st->cx = cx;
    st->cy = cy;
    st->th2 = (float)(px_th * px_th);
    st->n = m;
    st->bad = bad;
    st->stop = bad || m < kAbsMinRows;
    st->best_count = 0;
    st->n_all = n;
    st->row0 = pr.row0;
    st->row32 = pr.row0 - B.base;
  }
}

// Hypotheses first .. first + count - 1.  models [count * 4][12] fp64 (centred frame), counts [count * 4] (-1: no pose).
__global__ void __launch_bounds__(kAbsThreads, 1) abs_round_kernel(const AbsState* __restrict__ st_all,
                                                                   const AbsRow32* __restrict__ rows32_all,
                                                                   const double* __restrict__ rows_all, int stride,
                                                                   int first, int count, unsigned long long seed,
                                                                   int ignore_stop, double* __restrict__ models_all,
                                                                   int* __restrict__ counts_all) {
  constexpr int NM = kAbsHypPerBlock * kAbsSlots, PW = NM / 8;   // models per block, per warp
  __shared__ AbsRow32 s_rows[kAbsTile];
  __shared__ float s_model[NM][12];
  __shared__ int s_valid[NM];
  const AbsState* st = st_all + blockIdx.y;
  if (!ignore_stop && st->stop) return;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const int n = st->n;
  const float th2 = st->th2;
  const double* rows = rows_all + st->row0 * stride;
  const AbsRow32* rows32 = rows32_all + st->row32;
  double* models = models_all + blockIdx.y * kAbsModels;
  int* counts = counts_all + blockIdx.y * kAbsCounts;
  if (tid < kAbsHypPerBlock) {
    const int local = blockIdx.x * kAbsHypPerBlock + tid;
    const AbsState S = *st;
    double out[kAbsSlots][12];
    int nm = 0;
    int idx[kAbsSample];
    if (local < count && draw_sample<kAbsSample>(seed, first + local, n, idx)) {
      double j[3][3], X[3][3];
#pragma unroll
      for (int k = 0; k < 3; ++k) abs_row64(S, rows + (size_t)idx[k] * stride, j[k], X[k]);
      nm = solve_p3p(j, X, out);
    }
    for (int k = 0; k < kAbsSlots; ++k) {
      const int slot = tid * kAbsSlots + k;
      s_valid[slot] = k < nm;
      if (k < nm) abs_proj32(S, out[k], s_model[slot]);
      for (int e = 0; e < 12; ++e)
        if (local < count) models[((size_t)local * kAbsSlots + k) * 12 + e] = k < nm ? out[k][e] : 0.0;
    }
  }
  int cnt[PW];
#pragma unroll
  for (int j = 0; j < PW; ++j) cnt[j] = 0;
  for (int t0 = 0; t0 < n; t0 += kAbsTile) {
    const int tn = min(kAbsTile, n - t0);
    __syncthreads();
    for (int r = tid; r < tn; r += kAbsThreads) s_rows[r] = rows32[t0 + r];
    __syncthreads();
#pragma unroll
    for (int j = 0; j < PW; ++j) {
      const int mi = wid + 8 * j;
      if (!s_valid[mi]) continue;
      float p[12];
#pragma unroll
      for (int e = 0; e < 12; ++e) p[e] = s_model[mi][e];
      for (int r0 = 0; r0 < tn; r0 += 32) {
        const int r = r0 + lane;
        const bool in = r < tn && abs_inlier(p, s_rows[r < tn ? r : 0], th2);
        cnt[j] += __popc(__ballot_sync(0xffffffffu, in));
      }
    }
  }
  if (lane == 0) {
#pragma unroll
    for (int j = 0; j < PW; ++j) {
      const int mi = wid + 8 * j;
      const int local = blockIdx.x * kAbsHypPerBlock + mi / kAbsSlots;
      if (local < count) counts[(size_t)blockIdx.x * NM + mi] = s_valid[mi] ? cnt[j] : -1;
    }
  }
}

__global__ void __launch_bounds__(1024) abs_select_kernel(AbsState* __restrict__ st, const double* __restrict__ models,
                                                          const int* __restrict__ counts, int nm, int done, double conf,
                                                          int max_iters) {
  select_round<12>(st + blockIdx.y, models + blockIdx.y * kAbsModels, counts + blockIdx.y * kAbsCounts, nm, done,
                   kAbsSample, conf, max_iters);
}

// R <- exp([w]x) R (Rodrigues), t <- t + dt.
__device__ void pose_update(const double* m, const double* w, const double* dt, double* out) {
  const double th2 = w[0] * w[0] + w[1] * w[1] + w[2] * w[2];
  double a, b;
  if (th2 < 1e-12) {
    a = 1.0 - th2 / 6.0;
    b = 0.5 - th2 / 24.0;
  } else {
    const double th = sqrt(th2);
    a = sin(th) / th;
    b = (1.0 - cos(th)) / th2;
  }
  const double K[9] = {0.0, -w[2], w[1], w[2], 0.0, -w[0], -w[1], w[0], 0.0};
  double E[9];
  for (int i = 0; i < 3; ++i)
    for (int k = 0; k < 3; ++k) {
      const double kk = K[3 * i] * K[k] + K[3 * i + 1] * K[3 + k] + K[3 * i + 2] * K[6 + k];
      E[3 * i + k] = (i == k ? 1.0 : 0.0) + a * K[3 * i + k] + b * kk;
    }
  for (int i = 0; i < 3; ++i)
    for (int k = 0; k < 3; ++k) out[3 * i + k] = E[3 * i] * m[k] + E[3 * i + 1] * m[3 + k] + E[3 * i + 2] * m[6 + k];
  for (int i = 0; i < 3; ++i) out[9 + i] = m[9 + i] + dt[i];
}

// Solve the 6x6 normal equations (upper triangle h[21] row by row, g[6]) by Cholesky.  False unless positive definite.
__device__ bool solve6(const double* h, const double* g, double* x) {
  double L[6][6];
  int e = 0;
  for (int i = 0; i < 6; ++i)
    for (int j = i; j < 6; ++j) L[j][i] = h[e++];
  for (int j = 0; j < 6; ++j) {
    double s = L[j][j];
    for (int k = 0; k < j; ++k) s -= L[j][k] * L[j][k];
    if (!(s > 0.0)) return false;
    L[j][j] = sqrt(s);
    for (int i = j + 1; i < 6; ++i) {
      double v = L[i][j];
      for (int k = 0; k < j; ++k) v -= L[i][k] * L[j][k];
      L[i][j] = v / L[j][j];
    }
  }
  double y[6];
  for (int i = 0; i < 6; ++i) {
    double v = g[i];
    for (int k = 0; k < i; ++k) v -= L[i][k] * y[k];
    y[i] = v / L[i][i];
  }
  for (int i = 5; i >= 0; --i) {
    double v = y[i];
    for (int k = i + 1; k < 6; ++k) v -= L[k][i] * x[k];
    x[i] = v / L[i][i];
  }
  return true;
}

// Local optimisation + outputs.  Each refit runs kAbsGnSteps Gauss-Newton steps on the squared reprojection error over
// the inliers of the current pose (left-multiplied rotation update through the exponential map, translation added);
// the refit is kept while it has strictly more inliers.  Query q writes Rt_out[12 q ..] in world coordinates (NaN
// without a model), count_out[q] (-1: a value is not finite) and mask_out[row0 .. row0 + n_all).
__global__ void __launch_bounds__(kAbsLoThreads, 1) abs_lo_kernel(const AbsState* __restrict__ st_all,
                                                                  const AbsRow32* __restrict__ rows32_all,
                                                                  const double* __restrict__ rows_all, int stride,
                                                                  double* __restrict__ Rt_out,
                                                                  uint8_t* __restrict__ mask_out,
                                                                  int* __restrict__ count_out) {
  __shared__ double s_red[kAbsLoThreads / 32][27];
  __shared__ double s_cur[12], s_cand[12];
  __shared__ float s_p[12], s_pc[12];
  __shared__ int s_cnt[kAbsLoThreads / 32], s_ok;
  const AbsState* st = st_all + blockIdx.y;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const AbsState S = *st;
  const int n = S.n, n_all = S.n_all;
  const double* rows = rows_all + S.row0 * stride;
  const AbsRow32* rows32 = rows32_all + S.row32;
  int cur_count = S.bad ? 0 : S.best_count;
  if (tid < 12) s_cur[tid] = S.best[tid];
  __syncthreads();

  auto count_inliers = [&](const double* m64) -> int {    // block-wide, fixed order
    if (tid == 0) abs_proj32(S, m64, s_pc);
    __syncthreads();
    float p[12];
#pragma unroll
    for (int e = 0; e < 12; ++e) p[e] = s_pc[e];
    int c = 0;
    for (int r = tid; r < n; r += kAbsLoThreads) c += abs_inlier(p, rows32[r], S.th2);
    for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
    if (lane == 0) s_cnt[wid] = c;
    __syncthreads();
    int tot = 0;
    for (int w = 0; w < kAbsLoThreads / 32; ++w) tot += s_cnt[w];
    __syncthreads();
    return tot;
  };

  for (int it = 0; it < kAbsLoIters && cur_count >= kAbsMinRows; ++it) {
    if (tid == 0) abs_proj32(S, s_cur, s_p);
    if (tid < 12) s_cand[tid] = s_cur[tid];
    __syncthreads();
    float p[12];
#pragma unroll
    for (int e = 0; e < 12; ++e) p[e] = s_p[e];
    for (int g = 0; g < kAbsGnSteps; ++g) {
      double m[12];
#pragma unroll
      for (int e = 0; e < 12; ++e) m[e] = s_cand[e];
      double acc[27];
#pragma unroll
      for (int e = 0; e < 27; ++e) acc[e] = 0.0;
      for (int r = tid; r < n; r += kAbsLoThreads) {
        if (!abs_inlier(p, rows32[r], S.th2)) continue;
        const double* row = rows + (size_t)r * stride;
        double X[3], P[3];
        for (int i = 0; i < 3; ++i) X[i] = row[2 + i] - S.mean[i];
        for (int i = 0; i < 3; ++i) P[i] = m[3 * i] * X[0] + m[3 * i + 1] * X[1] + m[3 * i + 2] * X[2];
        const double x = P[0] + m[9], y = P[1] + m[10], z = P[2] + m[11];
        if (!(z > 0.0)) continue;
        const double iz = 1.0 / z;
        const double ru = S.fx * x * iz + S.cx - row[0], rv = S.fy * y * iz + S.cy - row[1];
        // d(x, y, z) / d(w, dt) = [-[P]x | I]; projection Jacobian [[fx/z, 0, -fx x/z^2], [0, fy/z, -fy y/z^2]]
        const double pu[3] = {S.fx * iz, 0.0, -S.fx * x * iz * iz}, pv[3] = {0.0, S.fy * iz, -S.fy * y * iz * iz};
        const double nPx[3][3] = {{0.0, P[2], -P[1]}, {-P[2], 0.0, P[0]}, {P[1], -P[0], 0.0}};   // -[P]x
        double ju[6], jv[6];
        for (int c = 0; c < 3; ++c) {
          ju[c] = pu[0] * nPx[0][c] + pu[1] * nPx[1][c] + pu[2] * nPx[2][c];
          jv[c] = pv[0] * nPx[0][c] + pv[1] * nPx[1][c] + pv[2] * nPx[2][c];
          ju[3 + c] = pu[c];
          jv[3 + c] = pv[c];
        }
        int e = 0;
#pragma unroll
        for (int i = 0; i < 6; ++i)
#pragma unroll
          for (int k = i; k < 6; ++k) acc[e++] += ju[i] * ju[k] + jv[i] * jv[k];
#pragma unroll
        for (int i = 0; i < 6; ++i) acc[21 + i] += ju[i] * ru + jv[i] * rv;
      }
#pragma unroll
      for (int e = 0; e < 27; ++e) {
        const double v = warp_sum_d(acc[e]);
        if (lane == 0) s_red[wid][e] = v;
      }
      __syncthreads();
      if (tid == 0) {
        double hg[27], dx[6];
        for (int e = 0; e < 27; ++e) {
          double v = 0.0;
          for (int w = 0; w < kAbsLoThreads / 32; ++w) v += s_red[w][e];
          hg[e] = v;
        }
        s_ok = solve6(hg, hg + 21, dx);
        if (s_ok) {
          const double w[3] = {-dx[0], -dx[1], -dx[2]}, dt[3] = {-dx[3], -dx[4], -dx[5]};
          double nm[12];
          pose_update(m, w, dt, nm);
          for (int e = 0; e < 12; ++e) s_ok &= isfinite(nm[e]);
          if (s_ok)
            for (int e = 0; e < 12; ++e) s_cand[e] = nm[e];
        }
      }
      __syncthreads();
      if (!s_ok) break;
    }
    if (!s_ok) break;
    const int c = count_inliers(s_cand);
    if (c <= cur_count) break;
    cur_count = c;
    if (tid < 12) s_cur[tid] = s_cand[tid];
    __syncthreads();
  }

  if (tid == 0) {
    const double nan = __longlong_as_double(0x7ff8000000000000ll);
    const bool has = cur_count > 0;
    for (int i = 0; i < 9; ++i) Rt_out[12 * blockIdx.y + i] = has ? s_cur[i] : nan;
    for (int i = 0; i < 3; ++i)          // x = R (X - c) + t = R X + (t - R c)
      Rt_out[12 * blockIdx.y + 9 + i] =
          has ? s_cur[9 + i] - (s_cur[3 * i] * S.mean[0] + s_cur[3 * i + 1] * S.mean[1] + s_cur[3 * i + 2] * S.mean[2])
              : nan;
    count_out[blockIdx.y] = S.bad ? -1 : cur_count;
    abs_proj32(S, s_cur, s_p);
  }
  __syncthreads();
  float p[12];
#pragma unroll
  for (int e = 0; e < 12; ++e) p[e] = s_p[e];
  uint8_t* mask = mask_out + S.row0;
  for (int r = tid; r < n_all; r += kAbsLoThreads) mask[r] = cur_count > 0 && r < n && abs_inlier(p, rows32[r], S.th2);
}

// ---- the scan lift ------------------------------------------------------------------------------------------------
// torch.nn.functional.grid_sample(align_corners=True) of one channel at pixel (ix, iy), bilinear: the in-bounds
// corners nw, ne, sw, se in that order, weights and sums rounded one operation at a time (no fused multiply-add).
__device__ __forceinline__ double bilinear(const double* scan, int H, int W, int c, double ix, double iy) {
  const double x0 = floor(ix), y0 = floor(iy), x1 = x0 + 1.0, y1 = y0 + 1.0;
  const double w[4] = {__dmul_rn(__dsub_rn(x1, ix), __dsub_rn(y1, iy)), __dmul_rn(__dsub_rn(ix, x0), __dsub_rn(y1, iy)),
                       __dmul_rn(__dsub_rn(x1, ix), __dsub_rn(iy, y0)), __dmul_rn(__dsub_rn(ix, x0), __dsub_rn(iy, y0))};
  const double xs[4] = {x0, x1, x0, x1}, ys[4] = {y0, y0, y1, y1};
  double v = 0.0;
  for (int k = 0; k < 4; ++k)
    if (xs[k] >= 0.0 && xs[k] < (double)W && ys[k] >= 0.0 && ys[k] < (double)H)
      v = __dadd_rn(v, __dmul_rn(scan[((size_t)ys[k] * W + (size_t)xs[k]) * 3 + c], w[k]));
  return v;
}

// One block: matches m < count in order, kept rows appended at the query's running count (a block-wide prefix sum per
// 1024 matches keeps the match order).  A = the 3x4 top of the alignment, row-major.
struct LiftArgs {
  double A[12];
};
__global__ void __launch_bounds__(kLiftThreads) lift_scan_kernel(const double* __restrict__ scan, int H, int W,
                                                                 LiftArgs a, const double* __restrict__ matches,
                                                                 int mstride, int n, const double* __restrict__ n_dev,
                                                                 double* __restrict__ rows_out, int ostride,
                                                                 long long cap, double* __restrict__ count_dev) {
  __shared__ int s_warp[kLiftThreads / 32];
  __shared__ long long s_base;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  int m = n;
  if (n_dev != nullptr) {
    const double v = *n_dev;
    if (v >= 0.0 && v < (double)n) m = (int)v;
  }
  if (tid == 0) s_base = (long long)*count_dev;
  __syncthreads();
  for (int c0 = 0; c0 < m; c0 += kLiftThreads) {
    const int r = c0 + tid;
    bool keep = false;
    double out[5];
    if (r < m) {
      const double* p = matches + (size_t)r * mstride;
      const double ix = p[2], iy = p[3];
      if (ix >= 0.0 && ix <= (double)(W - 1) && iy >= 0.0 && iy <= (double)(H - 1)) {
        const size_t nn = ((size_t)rint(iy) * W + (size_t)rint(ix)) * 3;
        double X[3];
        keep = true;
        for (int c = 0; c < 3; ++c) {
          const double l = bilinear(scan, H, W, c, ix, iy);
          X[c] = isnan(l) ? scan[nn + c] : l;
          keep &= isfinite(X[c]);
        }
        out[0] = p[0];
        out[1] = p[1];
        for (int i = 0; i < 3; ++i)
          out[2 + i] = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(a.A[4 * i], X[0]), __dmul_rn(a.A[4 * i + 1], X[1])),
                                           __dmul_rn(a.A[4 * i + 2], X[2])),
                                 a.A[4 * i + 3]);
      }
    }
    const unsigned bal = __ballot_sync(0xffffffffu, keep);
    if (lane == 0) s_warp[wid] = __popc(bal);
    __syncthreads();
    int before = 0, total = 0;
    for (int w = 0; w < kLiftThreads / 32; ++w) {
      before += w < wid ? s_warp[w] : 0;
      total += s_warp[w];
    }
    const long long pos = s_base + before + __popc(bal & ((1u << lane) - 1u));
    if (keep && pos < cap)
      for (int k = 0; k < 5; ++k) rows_out[(size_t)pos * ostride + k] = out[k];
    __syncthreads();
    if (tid == 0) s_base = min(cap, s_base + total);
    __syncthreads();
  }
  if (tid == 0) *count_dev = (double)s_base;
}

struct AbsScratch {
  AbsState* st;
  AbsRow32* rows32;
  double* models;
  int* counts;
};

AbsScratch abs_carve(void* base, int queries, long long rows) {
  char* p = (char*)base;
  AbsScratch s;
  s.st = (AbsState*)p;
  p += align_up((size_t)queries * sizeof(AbsState), 1024);
  s.rows32 = (AbsRow32*)p;
  p += align_up((size_t)rows * sizeof(AbsRow32) + 16, 1024);
  s.models = (double*)p;
  p += align_up((size_t)queries * kAbsModels * sizeof(double), 1024);
  s.counts = (int*)p;
  return s;
}

}  // namespace

size_t abspose_scratch_bytes(int queries, long long rows, bool rounds) {
  return align_up((size_t)queries * sizeof(AbsState), 1024) + align_up((size_t)rows * sizeof(AbsRow32) + 16, 1024) +
         (rounds ? align_up((size_t)queries * kAbsModels * sizeof(double), 1024) +
                       (size_t)queries * kAbsCounts * sizeof(int)
                 : 0);
}

int abspose_chunk_queries() {
  const size_t per = sizeof(AbsState) + kAbsModels * sizeof(double) + kAbsCounts * sizeof(int);
  return (int)std::min<size_t>(kMaxGridY, std::max<size_t>(1, kBatchScratchBudget / per));
}

int launch_find_absolute_pose(const PairBatch& B, const double* intr, double px_th, const double* px_th_dev,
                              double conf, int max_iters, unsigned long long seed, void* scratch, double* Rt_out,
                              uint8_t* mask_out, int* count_out, cudaStream_t st) {
  const AbsScratch s = abs_carve(scratch, B.pairs, B.total);
  abs_prep_kernel<<<dim3(1, B.pairs), 1024, 0, st>>>(B, intr, Cam4{}, px_th, px_th_dev, s.rows32, s.st);
  P2P_LAUNCH_OK();
  for (int first = 0; first < max_iters; first += kAbsRound) {
    const int count = min(kAbsRound, max_iters - first);
    abs_round_kernel<<<dim3(cdiv(count, kAbsHypPerBlock), B.pairs), kAbsThreads, 0, st>>>(
        s.st, s.rows32, B.rows, B.stride, first, count, seed, 0, s.models, s.counts);
    P2P_LAUNCH_OK();
    abs_select_kernel<<<dim3(1, B.pairs), 1024, 0, st>>>(s.st, s.models, s.counts, count * kAbsSlots, first + count,
                                                         conf, max_iters);
    P2P_LAUNCH_OK();
  }
  abs_lo_kernel<<<dim3(1, B.pairs), kAbsLoThreads, 0, st>>>(s.st, s.rows32, B.rows, B.stride, Rt_out, mask_out,
                                                            count_out);
  P2P_LAUNCH_OK();
  return 0;
}

int launch_test_absolute_pose_hypotheses(const double* rows, int stride, int n, const double* intr, double px_th,
                                         unsigned long long seed, int count, void* scratch, double* models_out,
                                         int* counts_out, cudaStream_t st) {
  const PairBatch B = single_pair(rows, stride, n, nullptr);
  const AbsScratch s = abs_carve(scratch, 1, n);
  abs_prep_kernel<<<1, 1024, 0, st>>>(B, nullptr, Cam4{intr[0], intr[1], intr[2], intr[3]}, px_th, nullptr, s.rows32,
                                      s.st);
  P2P_LAUNCH_OK();
  abs_round_kernel<<<dim3(cdiv(count, kAbsHypPerBlock), 1), kAbsThreads, 0, st>>>(s.st, s.rows32, rows, stride, 0,
                                                                                   count, seed, 1, models_out,
                                                                                   counts_out);
  P2P_LAUNCH_OK();
  return 0;
}

int launch_lift_scan(const double* scan, int H, int W, const double* align, const double* matches, int match_stride,
                     int n, const double* n_dev, double* rows_out, int row_stride, long long cap, double* count_dev,
                     cudaStream_t st) {
  LiftArgs a;
  for (int i = 0; i < 12; ++i) a.A[i] = align[i];
  lift_scan_kernel<<<1, kLiftThreads, 0, st>>>(scan, H, W, a, matches, match_stride, n, n_dev, rows_out, row_stride, cap,
                                               count_dev);
  P2P_LAUNCH_OK();
  return 0;
}

}  // namespace p2p
