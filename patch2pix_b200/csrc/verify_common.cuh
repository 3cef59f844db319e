// The RANSAC engine of verify.cu (F / H, kinds 0 and 1), degensac.cu (F with the DEGENSAC check: kind 0's launches plus
// the plane-and-parallax round, kind 2), pose.cu (E, kind 3) and abspose.cu (absolute pose, kind 4): the two-view
// state, the F / H minimal solvers, scoring, the prep / round / select / local-optimisation kernels and their launch
// sequence (find_model).  Each translation unit instantiates the kinds it launches; pose.cu and abspose.cu define
// Kind<3> and Kind<4> before they do.
//
// Every kernel serves a batch of pairs: pair p is blockIdx.y and owns the state st[p], its rows of the concatenated
// row array (st[p].row0 ..), its fp32 rows (rows32 + st[p].row32) and its round models / counts (kPairModels /
// kPairCounts per pair).  A pair's arithmetic does not depend on the other pairs.
#pragma once
#include <math.h>

#include <algorithm>

#include "kernels.h"
#include "ransac_common.cuh"

namespace p2p {
namespace {


constexpr int kRound = 1024;        // hypotheses per round
constexpr int kHypPerBlock = 8;     // hypotheses solved (one thread each) and scored per block
constexpr int kScoreThreads = 256;  // 8 warps
constexpr int kLoIters = 4;         // local-optimisation refits
constexpr int kLoThreads = 256;
constexpr int kDegenThreads = 256;  // records scan of one round: kRound * 3 slots over 256 threads
constexpr int kDegenMin = 5;        // a sample is H-degenerate when this many of its 7 points fit an induced H
constexpr unsigned long long kParallaxKey = 0x5851F42D4C957F2Dull;   // parallax draws use seed ^ kParallaxKey

struct VerifyState {
  double cx[2], cy[2], s[2];        // F / H: Hartley normalisation x' = s (x - c) of image 1 and image 2
  double best[9];                   // best model so far, in the scoring frame (pixels; E: camera coordinates)
  double plane[9];                  // DEGENSAC: H of the pending plane-and-parallax round, pixel coordinates
  int n;                            // effective row count
  int bad;                          // a coordinate is not finite
  int stop;                         // no further rounds are needed
  int best_count;                   // 0: no model yet
  int pending;                      // DEGENSAC: this round's records hold an H-degenerate sample
  int n_all;                        // rows of the pair (mask length)
  long long row0;                   // first row of the pair in the row array and the mask
  long long row32;                  // first row of the pair in rows32
  Intrinsics K;                     // E: the pair's cameras
  float th2;                        // squared inlier threshold in the scoring frame
};

// Pair p's cameras: intr[8 p ..] (device), or K1 for a single pair (intr == nullptr).
__device__ __forceinline__ Intrinsics pair_intrinsics(const double* intr, const Intrinsics& K1, int p) {
  if (intr == nullptr) return K1;
  const double* k = intr + 8 * (size_t)p;
  return Intrinsics{k[0], k[1], k[2], k[3], k[4], k[5], k[6], k[7]};
}

// Pixels -> camera coordinates, (p - c) / f per axis: a subtraction, then a division (fp64, correctly rounded).
__device__ __forceinline__ void to_camera(const double* p, const Intrinsics& K, double& x1, double& y1, double& x2,
                                          double& y2) {
  x1 = (p[0] - K.cx1) / K.fx1;
  y1 = (p[1] - K.cy1) / K.fy1;
  x2 = (p[2] - K.cx2) / K.fx2;
  y2 = (p[3] - K.cy2) / K.fy2;
}

// cv2.findEssentialMat's threshold in camera coordinates: px_th / ((fx + fy) / 2) of view 2, squared.
__device__ __forceinline__ float ess_th2(double px_th, const Intrinsics& K) {
  const double th = px_th / ((K.fx2 + K.fy2) / 2.0);
  return (float)(th * th);
}

// Row p in the solvers' frame: camera coordinates for E (kind 3), Hartley-normalised coordinates otherwise.
template <int KIND>
__device__ __forceinline__ void to_frame(const VerifyState& S, const double* p, double (&q)[4]) {
  if constexpr (KIND == 3) {
    to_camera(p, S.K, q[0], q[1], q[2], q[3]);
  } else {
    q[0] = (p[0] - S.cx[0]) * S.s[0];
    q[1] = (p[1] - S.cy[0]) * S.s[0];
    q[2] = (p[2] - S.cx[1]) * S.s[1];
    q[3] = (p[3] - S.cy[1]) * S.s[1];
  }
}

// ---- fp64 linear algebra (one thread) ----------------------------------------------------------------------------

__device__ __forceinline__ double det3(const double* m) {
  return m[0] * (m[4] * m[8] - m[5] * m[7]) - m[1] * (m[3] * m[8] - m[5] * m[6]) + m[2] * (m[3] * m[7] - m[4] * m[6]);
}

// Real roots of a3 l^3 + a2 l^2 + a1 l + a0 (trigonometric form for three real roots, Cardano for one).
__device__ int cubic_roots(double a3, double a2, double a1, double a0, double (&r)[3]) {
  const double m = fmax(fmax(fabs(a3), fabs(a2)), fmax(fabs(a1), fabs(a0)));
  if (!(m > 0.0)) return 0;
  if (fabs(a3) <= 1e-12 * m) {                        // degree drop: one root went to infinity
    if (fabs(a2) <= 1e-12 * m) {
      if (fabs(a1) <= 1e-12 * m) return 0;
      r[0] = -a0 / a1;
      return 1;
    }
    const double disc = a1 * a1 - 4.0 * a2 * a0;
    if (disc < 0.0) return 0;
    const double qq = -0.5 * (a1 + copysign(sqrt(disc), a1));
    r[0] = qq / a2;
    if (qq == 0.0) return 1;
    r[1] = a0 / qq;
    return 2;
  }
  const double b = a2 / a3, c = a1 / a3, d = a0 / a3;
  const double p = c - b * b / 3.0, q = 2.0 * b * b * b / 27.0 - b * c / 3.0 + d, shift = -b / 3.0;
  const double disc = q * q / 4.0 + p * p * p / 27.0;
  if (disc > 0.0) {
    const double sq = sqrt(disc);
    r[0] = cbrt(-q / 2.0 + sq) + cbrt(-q / 2.0 - sq) + shift;
    return 1;
  }
  if (p >= 0.0) {
    r[0] = shift;
    return 1;
  }
  const double rr = 2.0 * sqrt(-p / 3.0);
  const double phi = acos(fmin(1.0, fmax(-1.0, 1.5 * q / p * sqrt(-3.0 / p)))) / 3.0;
  for (int k = 0; k < 3; ++k) r[k] = rr * cos(phi - 2.0943951023931957 * k) + shift;
  return 3;
}

__device__ __forceinline__ void mat3_mul(const double* a, const double* b, double* c) {
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) c[i * 3 + j] = a[i * 3] * b[j] + a[i * 3 + 1] * b[3 + j] + a[i * 3 + 2] * b[6 + j];
}

// Normalised-coordinate model -> pixel coordinates.  F = T2^T Fn T1 scaled to unit Frobenius norm;
// H = T2^-1 Hn T1 scaled to H[2][2] = 1.  False when the scale is degenerate.
template <int KIND>
__device__ bool denormalise(const VerifyState& S, const double* mn, double* out) {
  const double T1[9] = {S.s[0], 0.0, -S.s[0] * S.cx[0], 0.0, S.s[0], -S.s[0] * S.cy[0], 0.0, 0.0, 1.0};
  double tmp[9];
  mat3_mul(mn, T1, tmp);
  if (KIND == 0) {
    const double T2t[9] = {S.s[1], 0.0, 0.0, 0.0, S.s[1], 0.0, -S.s[1] * S.cx[1], -S.s[1] * S.cy[1], 1.0};
    mat3_mul(T2t, tmp, out);
    double nrm = 0.0;
    for (int j = 0; j < 9; ++j) nrm += out[j] * out[j];
    if (!(nrm > 0.0)) return false;
    nrm = 1.0 / sqrt(nrm);
    for (int j = 0; j < 9; ++j) out[j] *= nrm;
    return true;
  }
  const double T2i[9] = {1.0 / S.s[1], 0.0, S.cx[1], 0.0, 1.0 / S.s[1], S.cy[1], 0.0, 0.0, 1.0};
  mat3_mul(T2i, tmp, out);
  double amax = 0.0;
  for (int j = 0; j < 9; ++j) amax = fmax(amax, fabs(out[j]));
  if (!(fabs(out[8]) > 1e-12 * amax)) return false;
  const double inv = 1.0 / out[8];
  for (int j = 0; j < 9; ++j) out[j] *= inv;
  out[8] = 1.0;
  return true;
}

// 7-point solver on normalised rows (x1, y1, x2, y2): up to 3 models x2^T F x1 = 0 in normalised coordinates,
// ordered by ascending lambda of det(lambda F1 + (1 - lambda) F2) = 0.
__device__ int solve_f7(const double (&p)[7][4], double (&out)[3][9]) {
  double A[7][9], N[2][9];
  for (int i = 0; i < 7; ++i) {
    const double x1 = p[i][0], y1 = p[i][1], x2 = p[i][2], y2 = p[i][3];
    const double row[9] = {x2 * x1, x2 * y1, x2, y2 * x1, y2 * y1, y2, x1, y1, 1.0};
    for (int j = 0; j < 9; ++j) A[i][j] = row[j];
  }
  if (!null_space<7>(A, N)) return 0;
  double D[9], M[9], v[4];
  for (int j = 0; j < 9; ++j) D[j] = N[0][j] - N[1][j];
  const double ls[4] = {0.0, 1.0, -1.0, 2.0};        // the cubic from its values at lambda = 0, 1, -1, 2
  for (int t = 0; t < 4; ++t) {
    for (int j = 0; j < 9; ++j) M[j] = N[1][j] + ls[t] * D[j];
    v[t] = det3(M);
  }
  const double a0 = v[0], a2 = 0.5 * (v[1] + v[2]) - v[0], odd = 0.5 * (v[1] - v[2]);
  const double a3 = (v[3] - v[0] - 4.0 * a2 - 2.0 * odd) / 6.0, a1 = odd - a3;
  double r[3];
  const int nr = cubic_roots(a3, a2, a1, a0, r);
  for (int k = 0; k < nr; ++k)
    for (int it = 0; it < 2; ++it) {                    // Newton polish
      const double l = r[k];
      const double f = ((a3 * l + a2) * l + a1) * l + a0, df = (3.0 * a3 * l + 2.0 * a2) * l + a1;
      if (df != 0.0) r[k] = l - f / df;
    }
  for (int i = 1; i < nr; ++i)
    for (int k = i; k > 0 && r[k] < r[k - 1]; --k) { const double t = r[k]; r[k] = r[k - 1]; r[k - 1] = t; }
  for (int k = 0; k < nr; ++k)
    for (int j = 0; j < 9; ++j) out[k][j] = N[1][j] + r[k] * D[j];
  return nr;
}

__device__ __forceinline__ double orient(double ax, double ay, double bx, double by, double cx, double cy) {
  return (bx - ax) * (cy - ay) - (by - ay) * (cx - ax);
}

// 4-point DLT on normalised rows.  Rejects a sample with 3 (near-)collinear points in either image, or whose
// triangle orientations do not agree between the images in the same way for all four triples.
__device__ int solve_h4(const double (&p)[4][4], double (&out)[1][9]) {
  const int tri[4][3] = {{0, 1, 2}, {0, 1, 3}, {0, 2, 3}, {1, 2, 3}};
  int sgn = 0;
  for (int t = 0; t < 4; ++t) {
    const int a = tri[t][0], b = tri[t][1], c = tri[t][2];
    const double o1 = orient(p[a][0], p[a][1], p[b][0], p[b][1], p[c][0], p[c][1]);
    const double o2 = orient(p[a][2], p[a][3], p[b][2], p[b][3], p[c][2], p[c][3]);
    if (!(fabs(o1) > 1e-6) || !(fabs(o2) > 1e-6)) return 0;
    const int s = (o1 > 0.0) == (o2 > 0.0) ? 1 : -1;
    if (t == 0) sgn = s;
    else if (s != sgn) return 0;
  }
  double A[8][9], N[1][9];
  for (int i = 0; i < 4; ++i) {
    const double x = p[i][0], y = p[i][1], u = p[i][2], v = p[i][3];
    const double r0[9] = {-x, -y, -1.0, 0.0, 0.0, 0.0, u * x, u * y, u};
    const double r1[9] = {0.0, 0.0, 0.0, -x, -y, -1.0, v * x, v * y, v};
    for (int j = 0; j < 9; ++j) { A[2 * i][j] = r0[j]; A[2 * i + 1][j] = r1[j]; }
  }
  if (!null_space<8>(A, N)) return 0;
  for (int j = 0; j < 9; ++j) out[0][j] = N[0][j];
  return 1;
}

// ---- scoring ------------------------------------------------------------------------------------------------------
// F: dd^2 / den < th^2.  H: |pi(H x1) - x2|^2 < th^2, never with a non-positive or vanishing third coordinate.
template <int KIND>
__device__ __forceinline__ bool is_inlier(const float* m, float4 r, float th2) {
  if (KIND == 0) {
    float dd, den;
    sampson_terms<float>(m, r.x, r.y, r.z, r.w, dd, den);
    return dd * dd < th2 * den;
  }
  const float w = m[6] * r.x + m[7] * r.y + m[8];
  const float u = m[0] * r.x + m[1] * r.y + m[2] - r.z * w, v = m[3] * r.x + m[4] * r.y + m[5] - r.w * w;
  return w > 1e-8f && u * u + v * v < th2 * w * w;
}

// ---- the kinds ----------------------------------------------------------------------------------------------------
// What the shared kernels take from Kind<KIND>, all fixed at compile time:
//   State, Row32           the pair state and the fp32 scoring row
//   kSample, kSlots        rows per minimal sample, up to kSlots models per sample
//   kPairSlots             model slots per hypothesis in a pair's round buffers (F's 3 for F, H and DEGENSAC, which
//                          share one scratch layout)
//   kModel                 doubles per model
//   kLoMin                 LO refits from kLoMin inliers
//   kTile                  rows staged in shared memory per scoring pass
//   kLoSteps, kLoSums      per LO refit, kLoSteps accumulate-and-solve steps over kLoSums per-row sums
//   prep                   launches the prep kernel (host)
//   image(S, m, e)         element e of a model's fp32 scoring image
//   inlier(m, r, th2)      the fp32 inlier test of scoring row r under an image m
//   solve_sample           a minimal sample's row indices -> models in the scoring frame
//   lo_row(S, c, p, acc)   adds row p's sums, linearised at the candidate c, to acc
//   lo_solve(S, c, red)    the per-warp sums red -> the next candidate (false: none)
//   write_model            the LO kernel's model output
// Kind 2 is DEGENSAC's plane-and-parallax round (F from 2 rows and H, no solver); kind 3, E, is defined in pose.cu and
// kind 4, absolute pose, in abspose.cu.
template <int KIND> struct Kind;

// What kinds 0 to 3 share: VerifyState, fp32 rows (x1, y1, x2, y2) in the scoring frame, models of 9 doubles scored
// through their fp32 cast, samples and LO rows mapped to the solvers' frame by to_frame, and one LO step per refit: the
// 45 sums of the normal matrix, its smallest eigenvector, then Kind<KIND>::refit.  Kind<KIND> adds kScore (the inlier
// test, 0: Sampson, F and E; 1: transfer error, H), solve (a minimal sample in the solvers' frame -> models in the
// scoring frame) and refit (the smallest eigenvector -> a model in the scoring frame, false: none).
template <int KIND> struct TwoView {
  using State = VerifyState;
  using Row32 = float4;
  static constexpr int kModel = 9, kLoSteps = 1, kLoSums = 45;
  static void prep(dim3 grid, cudaStream_t st, const PairBatch& B, const double* intr, const Intrinsics& K1,
                   double px_th, const double* px_th_dev, float4* rows32, VerifyState* s);
  static __device__ __forceinline__ float image(const VerifyState&, const double* m, int e) { return (float)m[e]; }
  static __device__ __forceinline__ bool inlier(const float* m, float4 r, float th2) {
    return is_inlier<Kind<KIND>::kScore>(m, r, th2);
  }
  template <int S, int SL>
  static __device__ __forceinline__ int solve_sample(const VerifyState& st, const double* rows, int stride,
                                                     const int (&idx)[S], double (&out)[SL][9]) {
    double p[S][4];
#pragma unroll
    for (int k = 0; k < S; ++k) to_frame<KIND>(st, rows + (size_t)idx[k] * stride, p[k]);
    return Kind<KIND>::solve(st, p, out);
  }
  static __device__ __forceinline__ void lo_row(const VerifyState& S, const double*, const double* p,
                                                double (&acc)[45]) {
    double q[4];
    to_frame<KIND>(S, p, q);
    const double x = q[0], y = q[1], u = q[2], v = q[3];
    if (Kind<KIND>::kScore == 0) {
      const double a[9] = {u * x, u * y, u, v * x, v * y, v, x, y, 1.0};
      int e = 0;
#pragma unroll
      for (int i = 0; i < 9; ++i)
#pragma unroll
        for (int j = i; j < 9; ++j) acc[e++] += a[i] * a[j];
    } else {
      const double a[9] = {-x, -y, -1.0, 0.0, 0.0, 0.0, u * x, u * y, u};
      const double b[9] = {0.0, 0.0, 0.0, -x, -y, -1.0, v * x, v * y, v};
      int e = 0;
#pragma unroll
      for (int i = 0; i < 9; ++i)
#pragma unroll
        for (int j = i; j < 9; ++j) acc[e++] += a[i] * a[j] + b[i] * b[j];
    }
  }
  static __device__ __forceinline__ bool lo_solve(const VerifyState& S, const double*, const double (*red)[45],
                                                  double* out) {
    double M[9][9], h[9];
    int e = 0;
    for (int i = 0; i < 9; ++i)
      for (int j = i; j < 9; ++j) {
        double v = 0.0;
        for (int w = 0; w < kLoThreads / 32; ++w) v += red[w][e];
        M[i][j] = M[j][i] = v;
        ++e;
      }
    jacobi_min_eigvec<9>(M, h);
    return Kind<KIND>::refit(S, h, out);
  }
  // The model, NaN when a row is not finite, zeros without a model.
  static __device__ __forceinline__ void write_model(const VerifyState&, const double* m, int count, int bad,
                                                     double* out) {
    const int t = threadIdx.x;
    if (t < 9) out[t] = bad ? __longlong_as_double(0x7ff8000000000000ll) : (count > 0 ? m[t] : 0.0);
  }
};

template <> struct Kind<0> : TwoView<0> {                          // F: 7-point, up to 3 roots
  static constexpr int kSample = 7, kSlots = 3, kPairSlots = 3, kLoMin = 8, kScore = 0, kTile = 2048;
  static __device__ int solve(const VerifyState& S, const double (&p)[7][4], double (&out)[3][9]) {
    double mn[3][9];
    const int raw = solve_f7(p, mn);
    int nm = 0;
    for (int k = 0; k < raw; ++k)
      if (denormalise<0>(S, mn[k], out[nm])) ++nm;
    return nm;
  }
  // Rank 2: F <- F (I - e e^T), e the smallest right singular vector.
  static __device__ bool refit(const VerifyState& S, double (&h)[9], double* out) {
    double G[3][3], ev[3];
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) G[i][j] = h[i] * h[j] + h[3 + i] * h[3 + j] + h[6 + i] * h[6 + j];
    jacobi_min_eigvec<3>(G, ev);
    for (int i = 0; i < 3; ++i) {
      const double fe = h[3 * i] * ev[0] + h[3 * i + 1] * ev[1] + h[3 * i + 2] * ev[2];
      for (int j = 0; j < 3; ++j) h[3 * i + j] -= fe * ev[j];
    }
    return denormalise<0>(S, h, out);
  }
};
template <> struct Kind<1> : TwoView<1> {                          // H: 4-point DLT
  static constexpr int kSample = 4, kSlots = 1, kPairSlots = 3, kLoMin = 4, kScore = 1, kTile = 2048;
  static __device__ int solve(const VerifyState& S, const double (&p)[4][4], double (&out)[1][9]) {
    double mn[1][9];
    return solve_h4(p, mn) && denormalise<1>(S, mn[0], out[0]);
  }
  static __device__ bool refit(const VerifyState& S, double (&h)[9], double* out) { return denormalise<1>(S, h, out); }
};
template <> struct Kind<2> : TwoView<2> {
  static constexpr int kSample = 2, kSlots = 1, kPairSlots = 3, kScore = 0, kTile = 2048;
};

template <int KIND>
constexpr size_t kPairModels = (size_t)kRound * Kind<KIND>::kPairSlots * Kind<KIND>::kModel;   // doubles per pair
template <int KIND> constexpr size_t kPairCounts = (size_t)kRound * Kind<KIND>::kPairSlots;       // ints per pair

// a x + b y + c with the rounding fixed as fma(a, x, b y) + c, so that the result does not depend on how the compiler
// schedules the products of an expression it also computes elsewhere (DEGENSAC's H x1 in the tests and the models).
__device__ __forceinline__ double affine2(double a, double b, double c, double x, double y) { return fma(a, x, b * y) + c; }

// fp64 one-sided transfer error of row p under the pixel H below th2 (never with (H x1)_z <= 1e-8): DEGENSAC's plane
// tests, in the form of the oracle's error so that both take the same decisions.
__device__ __forceinline__ bool h_inlier64(const double* H, const double* p, double th2) {
  const double w = affine2(H[6], H[7], H[8], p[0], p[1]);
  if (!(w > 1e-8)) return false;
  const double u = affine2(H[0], H[1], H[2], p[0], p[1]) / w - p[2], v = affine2(H[3], H[4], H[5], p[0], p[1]) / w - p[3];
  return u * u + v * v < th2;
}

__device__ __forceinline__ void cross3(const double* a, const double* b, double* c) {
  c[0] = a[1] * b[2] - a[2] * b[1];
  c[1] = a[2] * b[0] - a[0] * b[2];
  c[2] = a[0] * b[1] - a[1] * b[0];
}
__device__ __forceinline__ double dot3(const double* a, const double* b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }

// [e]x M for a 3x3 M (row-major).
__device__ __forceinline__ void skew_mul(const double* e, const double* M, double* out) {
  for (int j = 0; j < 3; ++j) {
    out[j] = -e[2] * M[3 + j] + e[1] * M[6 + j];
    out[3 + j] = e[2] * M[j] - e[0] * M[6 + j];
    out[6 + j] = -e[1] * M[j] + e[0] * M[3 + j];
  }
}

// ---- DEGENSAC plane-and-parallax models (verify_round_kernel<2>) ----------------------------------------------
// Plane-and-parallax model of hypothesis `hyp` of the parallax stream: two distinct rows that are not within h_th of
// S.plane (a rejected draw is re-drawn, at most kMaxDraws draws), e' = (H x_a x x'_a) x (H x_b x x'_b), F = [e']x H at
// unit Frobenius norm.  False without a model.
__device__ bool parallax_model(const VerifyState& S, const double* rows, int stride, unsigned long long seed, int hyp,
                               double h_th2, double* F) {
  const double* H = S.plane;
  const unsigned long long ps = seed ^ kParallaxKey;
  int idx[2], d = 0;
  for (int k = 0; k < 2; ++k)
    for (;;) {
      if (d >= kMaxDraws) return false;
      idx[k] = draw_index(ps, hyp, d++, S.n);
      if (k == 1 && idx[1] == idx[0]) continue;
      if (!h_inlier64(H, rows + (size_t)idx[k] * stride, h_th2)) break;
    }
  double l[2][3];
  for (int k = 0; k < 2; ++k) {
    const double* r = rows + (size_t)idx[k] * stride;
    const double hx[3] = {affine2(H[0], H[1], H[2], r[0], r[1]), affine2(H[3], H[4], H[5], r[0], r[1]),
                          affine2(H[6], H[7], H[8], r[0], r[1])};
    const double x2[3] = {r[2], r[3], 1.0};
    cross3(hx, x2, l[k]);
  }
  double e[3];
  cross3(l[0], l[1], e);
  if (!(sqrt(dot3(e, e)) > 1e-12 * sqrt(dot3(l[0], l[0]) * dot3(l[1], l[1])))) return false;
  skew_mul(e, H, F);
  double nrm = 0.0;
  for (int j = 0; j < 9; ++j) nrm += F[j] * F[j];
  nrm = sqrt(nrm);
  if (!(nrm > 0.0)) return false;
  for (int j = 0; j < 9; ++j) F[j] /= nrm;
  return true;
}

// ---- kernels ------------------------------------------------------------------------------------------------------
// Effective row count, finiteness, the solvers' frame (F / H: the Hartley normalisation; E, CAMERA: the pair's
// cameras), the scoring threshold, and the fp32 rows in the scoring frame (F / H: pixels; E: camera coordinates).  A
// pair with fewer than min_rows rows, or a non-finite one, runs no rounds.  px_th_dev (device, nullable): pair p's
// threshold is px_th_dev[p] instead of px_th.
template <bool CAMERA>
__global__ void __launch_bounds__(1024) verify_prep_kernel(PairBatch B, const double* __restrict__ intr, Intrinsics K1,
                                                           double px_th, const double* __restrict__ px_th_dev,
                                                           int min_rows, float4* __restrict__ rows32_all,
                                                           VerifyState* __restrict__ st_all) {
  __shared__ double red[33];
  __shared__ int s_n;
  const int tid = threadIdx.x;
  VerifyState* st = st_all + blockIdx.y;
  const PairRange pr = pair_range(B, blockIdx.y);
  const int n = pr.n, stride = B.stride;
  const double* rows = B.rows + pr.row0 * stride;
  float4* rows32 = rows32_all + (pr.row0 - B.base);
  const Intrinsics K = pair_intrinsics(intr, K1, blockIdx.y);
  if (tid == 0) s_n = effective_rows(B, blockIdx.y, n);
  __syncthreads();
  const int m = s_n;
  double sx[4] = {0.0, 0.0, 0.0, 0.0};
  int bad = 0;
  for (int r = tid; r < m; r += 1024) {
    const double* p = rows + (size_t)r * stride;
    double q[4] = {p[0], p[1], p[2], p[3]};
    bad |= !(isfinite(q[0]) && isfinite(q[1]) && isfinite(q[2]) && isfinite(q[3]));
    if constexpr (CAMERA) to_camera(p, K, q[0], q[1], q[2], q[3]);
    else for (int k = 0; k < 4; ++k) sx[k] += q[k];
    rows32[r] = make_float4((float)q[0], (float)q[1], (float)q[2], (float)q[3]);
  }
  bad = __syncthreads_or(bad);
  double mean[4], dist[2] = {0.0, 0.0};
  if constexpr (!CAMERA) {
    for (int k = 0; k < 4; ++k) mean[k] = block_sum_1024(sx[k], red) / (double)(m > 0 ? m : 1);
    if (!bad)
      for (int r = tid; r < m; r += 1024) {
        const double* p = rows + (size_t)r * stride;
        dist[0] += sqrt((p[0] - mean[0]) * (p[0] - mean[0]) + (p[1] - mean[1]) * (p[1] - mean[1]));
        dist[1] += sqrt((p[2] - mean[2]) * (p[2] - mean[2]) + (p[3] - mean[3]) * (p[3] - mean[3]));
      }
    for (int k = 0; k < 2; ++k) dist[k] = block_sum_1024(dist[k], red) / (double)(m > 0 ? m : 1);
  }
  if (tid == 0) {
    if (px_th_dev != nullptr) px_th = px_th_dev[blockIdx.y];
    if constexpr (CAMERA) {
      st->K = K;
      st->th2 = ess_th2(px_th, K);
    } else {
      for (int k = 0; k < 2; ++k) {
        st->cx[k] = mean[2 * k];
        st->cy[k] = mean[2 * k + 1];
        st->s[k] = dist[k] > 0.0 ? 1.4142135623730951 / dist[k] : 1.0;
      }
      st->th2 = (float)(px_th * px_th);
    }
    for (int j = 0; j < 9; ++j) st->best[j] = 0.0;
    st->n = m;
    st->bad = bad;
    st->stop = bad || m < min_rows;
    st->best_count = 0;
    st->pending = 0;
    st->n_all = n;
    st->row0 = pr.row0;
    st->row32 = pr.row0 - B.base;
  }
}

template <int KIND>
void TwoView<KIND>::prep(dim3 grid, cudaStream_t st, const PairBatch& B, const double* intr, const Intrinsics& K1,
                         double px_th, const double* px_th_dev, float4* rows32, VerifyState* s) {
  verify_prep_kernel<KIND == 3><<<grid, 1024, 0, st>>>(B, intr, K1, px_th, px_th_dev, Kind<KIND>::kSample, rows32, s);
}

// Hypotheses first .. first + count - 1.  models [count * slots][kModel] fp64 (scoring frame), counts [count * slots]
// (-1: no model in that slot).
template <int KIND>
__global__ void __launch_bounds__(kScoreThreads, 1)
    verify_round_kernel(const typename Kind<KIND>::State* __restrict__ st_all,
                        const typename Kind<KIND>::Row32* __restrict__ rows32_all, const double* __restrict__ rows_all,
                        int stride, int first, int count, unsigned long long seed, int ignore_stop, double h_th2,
                        double* __restrict__ models_all, int* __restrict__ counts_all) {
  using K = Kind<KIND>;
  constexpr int S = K::kSample, SL = K::kSlots, L = K::kModel, NM = kHypPerBlock * SL, kTile = K::kTile;
  __shared__ typename K::Row32 s_rows[kTile];
  __shared__ float s_model[NM][L];
  __shared__ int s_valid[NM];
  const typename K::State* st = st_all + blockIdx.y;
  if constexpr (KIND == 2) {
    if (!st->pending) return;
  } else if (!ignore_stop && st->stop) {
    return;
  }
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const int n = st->n;
  const float th2 = st->th2;
  const double* rows = rows_all + st->row0 * stride;
  const typename K::Row32* rows32 = rows32_all + st->row32;
  double* models = models_all + blockIdx.y * kPairModels<KIND>;
  int* counts = counts_all + blockIdx.y * kPairCounts<KIND>;
  if (tid < kHypPerBlock) {
    const int local = blockIdx.x * kHypPerBlock + tid;
    double out[SL][L];
    int nm = 0;
    if constexpr (KIND == 2) {
      if (local < count && parallax_model(*st, rows, stride, seed, first + local, h_th2, out[0])) nm = 1;
    } else if (local < count) {
      int idx[S];
      if (draw_sample<S>(seed, first + local, n, idx)) nm = K::solve_sample(*st, rows, stride, idx, out);
    }
    for (int k = 0; k < SL; ++k) {
      const int slot = tid * SL + k;
      s_valid[slot] = k < nm;
      if constexpr (L == 9) {                             // the image is a cast: zeros for an empty slot
        for (int j = 0; j < L; ++j) {
          s_model[slot][j] = k < nm ? K::image(*st, out[k], j) : 0.f;
          if (local < count) models[((size_t)local * SL + k) * L + j] = k < nm ? out[k][j] : 0.0;
        }
      } else {
        // Images of the slots that hold a model only (scoring skips the others).  Behind a select, ptxas computes
        // every slot's image first: kind 4 then needs 217 registers and runs one block per SM instead of two.
        if (k < nm)
          for (int j = 0; j < L; ++j) s_model[slot][j] = K::image(*st, out[k], j);
        if (local < count)
          for (int j = 0; j < L; ++j) models[((size_t)local * SL + k) * L + j] = k < nm ? out[k][j] : 0.0;
      }
    }
  }
  int cnt[(NM + 7) / 8];
#pragma unroll
  for (int j = 0; j < (NM + 7) / 8; ++j) cnt[j] = 0;
  for (int t0 = 0; t0 < n; t0 += kTile) {
    const int tn = min(kTile, n - t0);
    __syncthreads();
    for (int r = tid; r < tn; r += kScoreThreads) s_rows[r] = rows32[t0 + r];
    __syncthreads();
#pragma unroll
    for (int j = 0; j < (NM + 7) / 8; ++j) {
      const int mi = wid + 8 * j;
      if (mi >= NM || !s_valid[mi]) continue;
      float m[L];
#pragma unroll
      for (int e = 0; e < L; ++e) m[e] = s_model[mi][e];
      for (int r0 = 0; r0 < tn; r0 += 32) {
        const int r = r0 + lane;
        const bool in = r < tn && K::inlier(m, s_rows[r < tn ? r : 0], th2);
        cnt[j] += __popc(__ballot_sync(0xffffffffu, in));
      }
    }
  }
  if (lane == 0) {
#pragma unroll
    for (int j = 0; j < (NM + 7) / 8; ++j) {
      const int mi = wid + 8 * j;
      const int local = blockIdx.x * kHypPerBlock + mi / SL;
      if (mi < NM && local < count) counts[(size_t)blockIdx.x * NM + mi] = s_valid[mi] ? cnt[j] : -1;
    }
  }
}

// Best of this round's nm models -> state if strictly better than the best so far; then the stopping bound for samples
// of `sample` rows.  Pair p's round models and counts start pair_slots * kRound slots after pair p - 1's; models hold
// L doubles each.
template <int L = 9, typename State>
__global__ void __launch_bounds__(1024) verify_select_kernel(State* __restrict__ st, const double* __restrict__ models,
                                                             const int* __restrict__ counts, int nm, int done, int sample,
                                                             int pair_slots, double conf, int max_iters) {
  const size_t slots = (size_t)blockIdx.y * kRound * pair_slots;
  select_round<L>(st + blockIdx.y, models + slots * L, counts + slots, nm, done, sample, conf, max_iters);
}

// Local optimisation + outputs.  Each refit runs kLoSteps steps on the inliers of the current model (F: 8-point with
// rank-2 enforcement; H: DLT; E: 8-point projected onto the essential manifold; absolute pose: Gauss-Newton), and is
// kept while it has strictly more inliers; then the kernel writes model, mask and count.  Pair p writes
// model_out[kModel p ..], count_out[p] and mask_out[row0 .. row0 + n_all).
template <int KIND>
__global__ void __launch_bounds__(kLoThreads, 1)
    verify_lo_kernel(const typename Kind<KIND>::State* __restrict__ st_all,
                     const typename Kind<KIND>::Row32* __restrict__ rows32_all, const double* __restrict__ rows_all,
                     int stride, double* __restrict__ model_out, uint8_t* __restrict__ mask_out,
                     int* __restrict__ count_out) {
  using K = Kind<KIND>;
  constexpr int L = K::kModel;
  __shared__ double s_red[kLoThreads / 32][K::kLoSums];
  __shared__ double s_cur[L], s_cand[L];
  __shared__ float s_f32[L];
  __shared__ int s_cnt[kLoThreads / 32], s_ok;
  const typename K::State* st = st_all + blockIdx.y;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const int n = st->n, bad = st->bad, n_all = st->n_all;
  const float th2 = st->th2;
  const double* rows = rows_all + st->row0 * stride;
  const typename K::Row32* rows32 = rows32_all + st->row32;
  model_out += L * blockIdx.y;
  count_out += blockIdx.y;
  mask_out += st->row0;
  int cur_count = bad ? 0 : st->best_count;
  if (tid < L) s_cur[tid] = st->best[tid];
  __syncthreads();

  auto count_inliers = [&](const double* m64) -> int {    // block-wide, fixed order
    if (tid < L) s_f32[tid] = K::image(*st, m64, tid);
    __syncthreads();
    float m[L];
#pragma unroll
    for (int e = 0; e < L; ++e) m[e] = s_f32[e];
    int c = 0;
    for (int r = tid; r < n; r += kLoThreads) c += K::inlier(m, rows32[r], th2);
    for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
    if (lane == 0) s_cnt[wid] = c;
    __syncthreads();
    int tot = 0;
    for (int w = 0; w < kLoThreads / 32; ++w) tot += s_cnt[w];
    __syncthreads();
    return tot;
  };

  for (int it = 0; it < kLoIters && cur_count >= K::kLoMin; ++it) {
    if (tid < L) s_f32[tid] = K::image(*st, s_cur, tid);
    __syncthreads();
    float m[L];
#pragma unroll
    for (int e = 0; e < L; ++e) m[e] = s_f32[e];
    const typename K::State S = *st;                      // the frame, in registers for the row loop
    for (int g = 0; g < K::kLoSteps; ++g) {
      double at[L];                                       // the model this step linearises at
#pragma unroll
      for (int e = 0; e < L; ++e) at[e] = g == 0 ? s_cur[e] : s_cand[e];
      double acc[K::kLoSums];
#pragma unroll
      for (int e = 0; e < K::kLoSums; ++e) acc[e] = 0.0;
      for (int r = tid; r < n; r += kLoThreads)
        if (K::inlier(m, rows32[r], th2)) K::lo_row(S, at, rows + (size_t)r * stride, acc);
#pragma unroll
      for (int e = 0; e < K::kLoSums; ++e) {
        const double v = warp_sum_d(acc[e]);
        if (lane == 0) s_red[wid][e] = v;
      }
      __syncthreads();
      if (tid == 0) s_ok = K::lo_solve(S, at, s_red, s_cand);
      __syncthreads();
      if (!s_ok) break;
    }
    if (!s_ok) break;
    const int c = count_inliers(s_cand);
    if (c <= cur_count) break;
    cur_count = c;
    if (tid < L) s_cur[tid] = s_cand[tid];
    __syncthreads();
  }

  K::write_model(*st, s_cur, cur_count, bad, model_out);
  if (tid == 0) *count_out = bad ? -1 : cur_count;
  if (tid < L) s_f32[tid] = K::image(*st, s_cur, tid);
  __syncthreads();
  float m[L];
#pragma unroll
  for (int e = 0; e < L; ++e) m[e] = s_f32[e];
  for (int r = tid; r < n_all; r += kLoThreads)
    mask_out[r] = cur_count > 0 && r < n && K::inlier(m, rows32[r], th2);
}

template <typename State, typename Row32>
struct Scratch {
  State* st;
  Row32* rows32;
  double* models;
  int* counts;
};

// `pairs` states, `rows` fp32 rows, then nhyp hypotheses' models and counts per pair (nhyp = kRound: pair strides
// kPairModels / kPairCounts).
template <int KIND>
Scratch<typename Kind<KIND>::State, typename Kind<KIND>::Row32> carve(void* base, int pairs, long long rows, int nhyp) {
  using K = Kind<KIND>;
  char* p = (char*)base;
  Scratch<typename K::State, typename K::Row32> s;
  s.st = (typename K::State*)p;
  p += align_up((size_t)pairs * sizeof(typename K::State), 1024);
  s.rows32 = (typename K::Row32*)p;
  p += align_up((size_t)rows * sizeof(typename K::Row32) + 16, 1024);
  s.models = (double*)p;
  p += align_up((size_t)pairs * nhyp * K::kPairSlots * K::kModel * sizeof(double), 1024);
  s.counts = (int*)p;
  return s;
}

// Bytes carve<KIND> lays out for nhyp = kRound (rounds) or 0.
template <int KIND>
size_t scratch_bytes(int pairs, long long rows, bool rounds) {
  using K = Kind<KIND>;
  return align_up((size_t)pairs * sizeof(typename K::State), 1024) +
         align_up((size_t)rows * sizeof(typename K::Row32) + 16, 1024) +
         (rounds ? align_up((size_t)pairs * kPairModels<KIND> * sizeof(double), 1024) +
                       (size_t)pairs * kPairCounts<KIND> * sizeof(int)
                 : 0);
}

// Pairs per launch within kBatchScratchBudget.
template <int KIND>
int chunk_pairs() {
  const size_t per_pair = sizeof(typename Kind<KIND>::State) + kPairModels<KIND> * sizeof(double) +
                          kPairCounts<KIND> * sizeof(int);
  return (int)std::min<size_t>(kMaxGridY, std::max<size_t>(1, kBatchScratchBudget / per_pair));
}

template <int KIND, typename Scr>
int enqueue_round(const Scr& s, const PairBatch& B, int first, int count, unsigned long long seed, int ignore_stop,
                  cudaStream_t st, double h_th2 = 0.0) {
  verify_round_kernel<KIND><<<dim3(cdiv(count, kHypPerBlock), B.pairs), kScoreThreads, 0, st>>>(
      s.st, s.rows32, B.rows, B.stride, first, count, seed, ignore_stop, h_th2, s.models, s.counts);
  P2P_LAUNCH_OK();
  return 0;
}

// RANSAC for F (kind 0), H (1), E (3) or absolute pose (4): prep, then per round of kRound hypotheses a round and a
// select, then LO.  intr / K1: the pairs' cameras for E and absolute pose, as launch_find_essential and
// launch_find_absolute_pose take them; F and H ignore them.  px_th_dev (device, nullable): one threshold per pair of
// the launch, in place of px_th.
template <int KIND>
int find_model(const PairBatch& B, const double* intr, const Intrinsics& K1, double px_th, const double* px_th_dev,
               double conf, int max_iters, unsigned long long seed, void* scratch, double* model_out, uint8_t* mask_out,
               int* count_out, cudaStream_t st) {
  using K = Kind<KIND>;
  const auto s = carve<KIND>(scratch, B.pairs, B.total, kRound);
  K::prep(dim3(1, B.pairs), st, B, intr, K1, px_th, px_th_dev, s.rows32, s.st);
  P2P_LAUNCH_OK();
  for (int first = 0; first < max_iters; first += kRound) {
    const int count = min(kRound, max_iters - first);
    int rc = enqueue_round<KIND>(s, B, first, count, seed, 0, st);
    if (rc) return rc;
    verify_select_kernel<K::kModel><<<dim3(1, B.pairs), 1024, 0, st>>>(s.st, s.models, s.counts, count * K::kSlots,
                                                                        first + count, K::kSample, K::kPairSlots, conf,
                                                                        max_iters);
    P2P_LAUNCH_OK();
  }
  verify_lo_kernel<KIND><<<dim3(1, B.pairs), kLoThreads, 0, st>>>(s.st, s.rows32, B.rows, B.stride, model_out, mask_out,
                                                                  count_out);
  P2P_LAUNCH_OK();
  return 0;
}

// Test hook: hypotheses 0 .. count-1 of a single pair without selection.
template <int KIND>
int test_hypotheses(const double* rows, int stride, int n, const Intrinsics& K, double px_th, unsigned long long seed,
                    int count, void* scratch, double* models_out, int* counts_out, cudaStream_t st) {
  const PairBatch B = single_pair(rows, stride, n, nullptr);
  auto s = carve<KIND>(scratch, 1, n, 0);
  s.models = models_out;
  s.counts = counts_out;
  Kind<KIND>::prep(dim3(1), st, B, nullptr, K, px_th, nullptr, s.rows32, s.st);
  P2P_LAUNCH_OK();
  return enqueue_round<KIND>(s, B, 0, count, seed, 1, st);
}

}  // namespace
}  // namespace p2p
