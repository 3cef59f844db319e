// Relative pose on the device: RANSAC for an essential matrix (5-point minimal solver) with local optimisation, and
// pose recovery from E (cv2.findEssentialMat(..., RANSAC) + cv2.recoverPose semantics, utils/eval/geometry.py:32-48).
//
// p2p_find_essential enqueues, with no host sync:
//   ess_prep_kernel     (1 block)  effective row count, finiteness, fp32 copy of the rows in camera coordinates
//   ess_round_kernel    (x rounds) kRound hypotheses: 5-point sample -> up to 10 models (one thread each), then every
//                                  (model, row) pair scored in fp32 (Sampson error) by warps over rows in shared memory
//   ess_select_kernel   (x rounds) best model so far and the stopping bound, as verify.cu (s = 5)
//   ess_lo_kernel       (1 block)  8-point refit on the winner's inliers projected onto the essential manifold while
//                                  the count grows, final E, mask and count
// p2p_recover_pose enqueues:
//   pose_decompose_kernel (1 thread)   SVD of E -> the four candidates [R1|t], [R2|t], [R1|-t], [R2|-t]
//   pose_count_kernel     (kPoseBlocks) linear triangulation of every masked row against each candidate, cheirality and
//                                      distance test -> one 4-bit code per row and per-block integer counts
//   pose_select_kernel    (1 block)   fixed-order sum of the counts, first best candidate, R, t, count, mask
// A batch of pairs runs the same launches with the pair as grid dimension y: one block per pair for the one-block
// kernels, cdiv(count, 8) x pairs for a round and kPoseBlocks x pairs for pose_count_kernel.  Pair p's intrinsics,
// threshold and row range live in its state, so a pair's arithmetic does not depend on the other pairs.
// No grid size depends on the device and every combine runs in a fixed order, so results are bit-reproducible.
#include <algorithm>

#include <math.h>

#include "kernels.h"
#include "ransac_common.cuh"

namespace p2p {
namespace {

constexpr int kRound = 1024;        // hypotheses per round
constexpr int kHypPerBlock = 8;     // hypotheses solved (one thread each) and scored per block
constexpr int kScoreThreads = 256;  // 8 warps
constexpr int kTile = 1024;         // rows staged in shared memory per pass (16 KB)
constexpr int kSample = 5;
constexpr int kSlots = 10;          // real roots of the degree-10 polynomial
constexpr int kLoMin = 8;
constexpr int kLoIters = 4;
constexpr int kLoThreads = 256;
constexpr int kBisect = 64;         // bisection steps per root
constexpr int kNewton = 2;          // guarded Newton steps per root
constexpr double kZMax = 1e6;       // roots are searched in (-kZMax, kZMax]
constexpr int kPoseBlocks = 256;
constexpr int kPoseThreads = 256;

struct EssState {
  double best[9];                   // best model so far, camera coordinates
  Intrinsics K;                     // the pair's cameras
  float th2;                        // squared inlier threshold in camera coordinates
  int n;                            // effective row count
  int bad;                          // a coordinate is not finite
  int stop;                         // no further rounds are needed
  int best_count;                   // 0: no model yet
  int n_all;                        // rows of the pair (mask length)
  long long row0;                   // first row of the pair in the row array and the mask
  long long row32;                  // first row of the pair in rows32
};

struct PoseState {
  double R[2][9], t[3];             // R1, R2 row-major, t = U[:, 2]
  Intrinsics K;                     // the pair's cameras
  int n;                            // effective row count
  int valid;                        // E was finite and non-zero
  int n_all;                        // rows of the pair (mask length)
  long long row0;                   // first row of the pair in the row array and the masks
  long long row32;                  // first row of the pair in the codes
};

constexpr size_t kPairModels = (size_t)kRound * kSlots * 9;   // round-model doubles per pair
constexpr size_t kPairCounts = (size_t)kRound * kSlots;       // round-count ints per pair

// ---- 5-point solver (one thread; restated in oracle/pose_oracle.py) ------------------------------------------------
// Monomials of degree <= 3 in (x, y, z): x^3 y^3 x^2y xy^2 x^2z x^2 y^2z y^2 xyz xy | xz^2 xz x yz^2 yz y z^3 z^2 z 1.
// Degree 2: x^2 xy xz y^2 yz z^2 x y z 1.  Degree 1: x y z 1.  The tables give the index of a product.
__constant__ int kMul11[4][4] = {{0, 1, 2, 6}, {1, 3, 4, 7}, {2, 4, 5, 8}, {6, 7, 8, 9}};
__constant__ int kMul21[10][4] = {{0, 2, 4, 5},   {2, 3, 8, 9},   {4, 8, 10, 11},  {3, 1, 6, 7},    {8, 6, 13, 14},
                                  {10, 13, 16, 17}, {5, 9, 11, 12}, {9, 7, 14, 15}, {11, 14, 17, 18}, {12, 15, 18, 19}};

__device__ __forceinline__ void mul11(const double* a, const double* b, double* out, double sgn) {   // out += sgn a b
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) out[kMul11[i][j]] += sgn * (a[i] * b[j]);
}
__device__ __forceinline__ void mul21(const double* a, const double* b, double* out, double sgn) {
#pragma unroll
  for (int i = 0; i < 10; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) out[kMul21[i][j]] += sgn * (a[i] * b[j]);
}

// Horner on ascending coefficients.
template <int N>
__device__ __forceinline__ double peval(const double (&p)[N], double z) {
  double v = p[N - 1];
#pragma unroll
  for (int i = N - 2; i >= 0; --i) v = v * z + p[i];
  return v;
}

template <int NA, int NB>
__device__ __forceinline__ void pmul_acc(const double (&a)[NA], const double (&b)[NB], double* out, double sgn) {
#pragma unroll
  for (int i = 0; i < NA; ++i)
#pragma unroll
    for (int j = 0; j < NB; ++j) out[i + j] += sgn * (a[i] * b[j]);
}

// Sturm chain: 11 polynomials of degree 10 .. 0, descending coefficients, chain[kOff[i] ..].
__device__ __forceinline__ int sturm_off(int i) { return i * 11 - i * (i - 1) / 2; }

__device__ int sign_changes(const double* chain, double z) {
  int cnt = 0;
  double last = 0.0;
  for (int i = 0; i < 11; ++i) {
    const double* p = chain + sturm_off(i);
    double v = p[0];
    for (int k = 1; k < 11 - i; ++k) v = v * z + p[k];
    const double s = v > 0.0 ? 1.0 : (v < 0.0 ? -1.0 : 0.0);
    cnt += s != 0.0 && last != 0.0 && s != last;
    if (s != 0.0) last = s;
  }
  return cnt;
}

__device__ __forceinline__ void scale_to_unit(double* p, int len) {
  double s = 0.0;
  for (int k = 0; k < len; ++k) s = fmax(s, fabs(p[k]));
  if (s > 0.0)
    for (int k = 0; k < len; ++k) p[k] /= s;
}

// Real roots of d (ascending, degree 10) in (-zb, zb], zb = min(Cauchy bound, kZMax), ascending.  The chain assumes
// every remainder has full degree; a sample where that fails yields no roots.  chain: 66 doubles of scratch (shared).
__device__ int real_roots(const double (&d)[11], double* chain, double (&z)[10]) {
  for (int k = 0; k < 11; ++k) chain[k] = d[10 - k];
  for (int k = 0; k < 10; ++k) chain[11 + k] = d[10 - k] * (double)(10 - k);
  scale_to_unit(chain, 11);
  scale_to_unit(chain + 11, 10);
  for (int i = 2; i < 11; ++i) {
    const double* a = chain + sturm_off(i - 2);          // length 13 - i
    const double* b = chain + sturm_off(i - 1);          // length 12 - i
    double* r = chain + sturm_off(i);                    // length 11 - i
    const int lb = 12 - i;
    const double q1 = a[0] / b[0];
    double t[11];
    for (int k = 0; k < lb; ++k) t[k] = a[k + 1] - q1 * (k + 1 < lb ? b[k + 1] : 0.0);
    const double q0 = t[0] / b[0];
    for (int k = 0; k < lb - 1; ++k) r[k] = -(t[k + 1] - q0 * b[k + 1]);
    scale_to_unit(r, lb - 1);
  }
  for (int i = 0; i < 11; ++i) {
    const double* p = chain + sturm_off(i);
    if (!(p[0] != 0.0)) return 0;
    for (int k = 0; k < 11 - i; ++k)
      if (!isfinite(p[k])) return 0;
  }
  double cb = 0.0;
  for (int k = 0; k < 10; ++k) cb = fmax(cb, fabs(d[k]) / fabs(d[10]));
  const double zb = fmin(1.0 + cb, kZMax);
  if (!isfinite(zb)) return 0;
  const int v_lo = sign_changes(chain, -zb);
  const int nr = v_lo - sign_changes(chain, zb);
  double dd[10];
  for (int k = 0; k < 10; ++k) dd[k] = d[k + 1] * (double)(k + 1);
  for (int k = 0; k < nr && k < 10; ++k) {
    double lo = -zb, hi = zb;
    for (int it = 0; it < kBisect; ++it) {
      const double mid = 0.5 * (lo + hi);
      if (v_lo - sign_changes(chain, mid) >= k + 1) hi = mid;
      else lo = mid;
    }
    double x = 0.5 * (lo + hi);
    const double w = hi - lo;
    for (int it = 0; it < kNewton; ++it) {
      const double f = peval(d, x), df = peval(dd, x);
      const double step = f / df;
      if (df != 0.0 && fabs(step) <= w) x -= step;
    }
    z[k] = x;
  }
  return nr < 10 ? nr : 10;
}

// <e> - z <f> of Nister's elimination: polynomials in z (ascending) multiplying x (deg 3), y (deg 3) and 1 (deg 4).
__device__ __forceinline__ void row_polys(const double* be, const double* bf, double (&px)[4], double (&py)[4],
                                          double (&pc)[5]) {
  px[0] = be[2]; px[1] = be[1] - bf[2]; px[2] = be[0] - bf[1]; px[3] = -bf[0];
  py[0] = be[5]; py[1] = be[4] - bf[5]; py[2] = be[3] - bf[4]; py[3] = -bf[3];
  pc[0] = be[9]; pc[1] = be[8] - bf[9]; pc[2] = be[7] - bf[8]; pc[3] = be[6] - bf[7]; pc[4] = -bf[6];
}

// 5-point solver on camera-coordinate rows (x1, y1, x2, y2): up to 10 essential matrices x2^T E x1 = 0 at unit
// Frobenius norm, ascending in z.  M is this thread's 10 x 20 elimination matrix in shared memory.
__device__ int solve_e5(const double (&p)[5][4], double (*M)[20], double (&out)[kSlots][9]) {
  double A[5][9], N[4][9];
  for (int i = 0; i < 5; ++i) {
    const double x1 = p[i][0], y1 = p[i][1], x2 = p[i][2], y2 = p[i][3];
    const double row[9] = {x2 * x1, x2 * y1, x2, y2 * x1, y2 * y1, y2, x1, y1, 1.0};
    for (int j = 0; j < 9; ++j) A[i][j] = row[j];
  }
  if (!null_space<5>(A, N)) return 0;
  // E = x X + y Y + z Z + W: entry j as a polynomial in (x, y, z, 1)
  double e[9][4];
#pragma unroll
  for (int j = 0; j < 9; ++j)
#pragma unroll
    for (int v = 0; v < 4; ++v) e[j][v] = N[v][j];
  // 10 cubic constraints: det E = 0, then 2 E E^T E - tr(E E^T) E = 0 row-major
  {
    double c[10];
    double* r = M[0];
    for (int k = 0; k < 20; ++k) r[k] = 0.0;
    const int cof[3][4] = {{4, 8, 5, 7}, {3, 8, 5, 6}, {3, 7, 4, 6}};
    const double sg[3] = {1.0, -1.0, 1.0};
#pragma unroll
    for (int i = 0; i < 3; ++i) {
#pragma unroll
      for (int k = 0; k < 10; ++k) c[k] = 0.0;
      mul11(e[cof[i][0]], e[cof[i][1]], c, 1.0);
      mul11(e[cof[i][2]], e[cof[i][3]], c, -1.0);
      mul21(c, e[i], r, sg[i]);
    }
  }
  {
    double eet[6][10], tr[10];
    const int sym[3][3] = {{0, 1, 2}, {1, 3, 4}, {2, 4, 5}};
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
      for (int j = i; j < 3; ++j) {
        double* o = eet[sym[i][j]];
#pragma unroll
        for (int k = 0; k < 10; ++k) o[k] = 0.0;
#pragma unroll
        for (int k = 0; k < 3; ++k) mul11(e[3 * i + k], e[3 * j + k], o, 1.0);
      }
#pragma unroll
    for (int k = 0; k < 10; ++k) tr[k] = eet[0][k] + eet[3][k] + eet[5][k];
#pragma unroll
    for (int i = 0; i < 3; ++i)
#pragma unroll
      for (int j = 0; j < 3; ++j) {
        double* r = M[1 + 3 * i + j];
#pragma unroll
        for (int k = 0; k < 20; ++k) r[k] = 0.0;
#pragma unroll
        for (int k = 0; k < 3; ++k) mul21(eet[sym[i][k]], e[3 * k + j], r, 2.0);
        mul21(tr, e[3 * i + j], r, -1.0);
      }
  }
  // Gauss-Jordan with partial pivoting: the 10 leading monomials in terms of the trailing 10
  double amax0 = 0.0;
  for (int i = 0; i < 10; ++i)
    for (int k = 0; k < 20; ++k) amax0 = fmax(amax0, fabs(M[i][k]));
  if (!(amax0 > 0.0)) return 0;
  for (int c = 0; c < 10; ++c) {
    int p_ = c;
    for (int i = c + 1; i < 10; ++i)
      if (fabs(M[i][c]) > fabs(M[p_][c])) p_ = i;
    if (!(fabs(M[p_][c]) > 1e-12 * amax0)) return 0;
    if (p_ != c)
      for (int k = 0; k < 20; ++k) { const double t = M[c][k]; M[c][k] = M[p_][k]; M[p_][k] = t; }
    const double piv = M[c][c];
    for (int k = 0; k < 20; ++k) M[c][k] /= piv;
    for (int i = 0; i < 10; ++i) {
      if (i == c) continue;
      const double f = M[i][c];
      for (int k = 0; k < 20; ++k) M[i][k] -= f * M[c][k];
    }
  }
  // <k> = <x^2 z> - z <x^2>, <l> = <y^2 z> - z <y^2>, <m> = <xyz> - z <xy>; det [k; l; m] (z) = 0 has degree 10
  double kx[4], ky[4], kc[5], lx[4], ly[4], lc[5], mx[4], my[4], mc[5];
  row_polys(M[4] + 10, M[5] + 10, kx, ky, kc);
  row_polys(M[6] + 10, M[7] + 10, lx, ly, lc);
  row_polys(M[8] + 10, M[9] + 10, mx, my, mc);
  double d[11];
  {
    double c1[8], c2[8], c3[7];
#pragma unroll
    for (int k = 0; k < 8; ++k) c1[k] = c2[k] = 0.0;
#pragma unroll
    for (int k = 0; k < 7; ++k) c3[k] = 0.0;
    pmul_acc(ly, mc, c1, 1.0);
    pmul_acc(lc, my, c1, -1.0);
    pmul_acc(lx, mc, c2, 1.0);
    pmul_acc(lc, mx, c2, -1.0);
    pmul_acc(lx, my, c3, 1.0);
    pmul_acc(ly, mx, c3, -1.0);
#pragma unroll
    for (int k = 0; k < 11; ++k) d[k] = 0.0;
    pmul_acc(kx, c1, d, 1.0);
    pmul_acc(ky, c2, d, -1.0);
    pmul_acc(kc, c3, d, 1.0);
  }
  double z[10];
  const int nr = real_roots(d, M[0], z);     // the Sturm chain reuses the elimination matrix
  int nm = 0;
  for (int r = 0; r < nr; ++r) {
    const double zr = z[r];
    const double B[3][3] = {{peval(kx, zr), peval(ky, zr), peval(kc, zr)},
                            {peval(lx, zr), peval(ly, zr), peval(lc, zr)},
                            {peval(mx, zr), peval(my, zr), peval(mc, zr)}};
    const int pr[3][2] = {{0, 1}, {0, 2}, {1, 2}};
    double v[3] = {0.0, 0.0, 0.0}, best = -1.0;
    for (int q = 0; q < 3; ++q) {
      const double* a = B[pr[q][0]];
      const double* b = B[pr[q][1]];
      const double cr[3] = {a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]};
      const double nn = cr[0] * cr[0] + cr[1] * cr[1] + cr[2] * cr[2];
      if (nn > best) { best = nn; v[0] = cr[0]; v[1] = cr[1]; v[2] = cr[2]; }
    }
    const double x = v[0] / v[2], y = v[1] / v[2];
    double E[9], nrm = 0.0;
    for (int j = 0; j < 9; ++j) {
      E[j] = x * N[0][j] + y * N[1][j] + zr * N[2][j] + N[3][j];
      nrm += E[j] * E[j];
    }
    nrm = sqrt(nrm);
    bool ok = true;
    for (int j = 0; j < 9; ++j) {
      E[j] /= nrm;
      ok &= isfinite(E[j]);
    }
    if (!ok) continue;
    for (int j = 0; j < 9; ++j) out[nm][j] = E[j];
    ++nm;
  }
  return nm;
}

// ---- 3x3 SVD (one-sided Jacobi, fp64): A = U diag(s) V^T, s descending, U[:, 2] = U[:, 0] x U[:, 1] ---------------
// False when A has rank below 2 or is not finite.
__device__ bool svd3(const double* A, double (&U)[3][3], double (&s)[3], double (&Vm)[3][3]) {
  double B[3][3];   // columns b_j = B[.][j]
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) {
      B[i][j] = A[3 * i + j];
      Vm[i][j] = i == j ? 1.0 : 0.0;
    }
  for (int sweep = 0; sweep < 30; ++sweep) {
    bool rotated = false;
    for (int p = 0; p < 2; ++p)
      for (int q = p + 1; q < 3; ++q) {
        double al = 0.0, be = 0.0, ga = 0.0;
        for (int i = 0; i < 3; ++i) {
          al += B[i][p] * B[i][p];
          be += B[i][q] * B[i][q];
          ga += B[i][p] * B[i][q];
        }
        if (!(fabs(ga) > 1e-15 * sqrt(al * be))) continue;
        rotated = true;
        const double zeta = (be - al) / (2.0 * ga);
        const double t = copysign(1.0, zeta) / (fabs(zeta) + sqrt(1.0 + zeta * zeta));
        const double c = 1.0 / sqrt(1.0 + t * t), sn = c * t;
        for (int i = 0; i < 3; ++i) {
          const double bp = B[i][p], bq = B[i][q];
          B[i][p] = c * bp - sn * bq;
          B[i][q] = sn * bp + c * bq;
          const double vp = Vm[i][p], vq = Vm[i][q];
          Vm[i][p] = c * vp - sn * vq;
          Vm[i][q] = sn * vp + c * vq;
        }
      }
    if (!rotated) break;
  }
  for (int j = 0; j < 3; ++j) s[j] = sqrt(B[0][j] * B[0][j] + B[1][j] * B[1][j] + B[2][j] * B[2][j]);
  for (int i = 1; i < 3; ++i)       // descending, stable
    for (int k = i; k > 0 && s[k] > s[k - 1]; --k) {
      const double ts = s[k]; s[k] = s[k - 1]; s[k - 1] = ts;
      for (int r = 0; r < 3; ++r) {
        double t = B[r][k]; B[r][k] = B[r][k - 1]; B[r][k - 1] = t;
        t = Vm[r][k]; Vm[r][k] = Vm[r][k - 1]; Vm[r][k - 1] = t;
      }
    }
  if (!(s[1] > 0.0) || !isfinite(s[0])) return false;
  for (int j = 0; j < 2; ++j)
    for (int i = 0; i < 3; ++i) U[i][j] = B[i][j] / s[j];
  U[0][2] = U[1][0] * U[2][1] - U[2][0] * U[1][1];
  U[1][2] = U[2][0] * U[0][1] - U[0][0] * U[2][1];
  U[2][2] = U[0][0] * U[1][1] - U[1][0] * U[0][1];
  return true;
}

__device__ __forceinline__ double det3m(const double (&m)[3][3]) {
  return m[0][0] * (m[1][1] * m[2][2] - m[1][2] * m[2][1]) - m[0][1] * (m[1][0] * m[2][2] - m[1][2] * m[2][0]) +
         m[0][2] * (m[1][0] * m[2][1] - m[1][1] * m[2][0]);
}

__device__ __forceinline__ bool is_inlier_e(const float* m, float4 r, float th2) {
  float dd, den;
  sampson_terms<float>(m, r.x, r.y, r.z, r.w, dd, den);
  return dd * dd < th2 * den;
}

__device__ __forceinline__ void to_camera(const double* p, const Intrinsics& K, double& x1, double& y1, double& x2,
                                          double& y2) {
  x1 = (p[0] - K.cx1) / K.fx1;
  y1 = (p[1] - K.cy1) / K.fy1;
  x2 = (p[2] - K.cx2) / K.fx2;
  y2 = (p[3] - K.cy2) / K.fy2;
}

__device__ __forceinline__ int effective_rows(int n, const double* n_dev) {
  int m = n;
  if (n_dev != nullptr) {
    const double v = *n_dev;
    if (v >= 0.0 && v < (double)n) m = (int)v;
  }
  return m;
}

// Pair p's cameras: intr[8 p ..] (device), or K1 for a single pair (intr == nullptr).
__device__ __forceinline__ Intrinsics pair_intrinsics(const double* intr, const Intrinsics& K1, int p) {
  if (intr == nullptr) return K1;
  const double* k = intr + 8 * (size_t)p;
  return Intrinsics{k[0], k[1], k[2], k[3], k[4], k[5], k[6], k[7]};
}

// cv2.findEssentialMat's threshold in camera coordinates: px_th / ((fx + fy) / 2) of view 2, squared.
__device__ __forceinline__ float ess_th2(double px_th, const Intrinsics& K) {
  const double th = px_th / ((K.fx2 + K.fy2) / 2.0);
  return (float)(th * th);
}

// ---- essential-matrix RANSAC kernels -------------------------------------------------------------------------------
__global__ void __launch_bounds__(1024) ess_prep_kernel(PairBatch B, const double* __restrict__ intr, Intrinsics K1,
                                                        double px_th, float4* __restrict__ rows32_all,
                                                        EssState* __restrict__ st_all) {
  __shared__ int s_n;
  const int tid = threadIdx.x, p = blockIdx.y;
  EssState* st = st_all + p;
  const PairRange pr = pair_range(B, p);
  const int n = pr.n, stride = B.stride;
  const double* rows = B.rows + pr.row0 * stride;
  float4* rows32 = rows32_all + (pr.row0 - B.base);
  const Intrinsics K = pair_intrinsics(intr, K1, p);
  if (tid == 0) s_n = effective_rows(n, B.n_dev == nullptr ? nullptr : B.n_dev + p);
  __syncthreads();
  const int m = s_n;
  int bad = 0;
  for (int r = tid; r < m; r += 1024) {
    const double* p = rows + (size_t)r * stride;
    bad |= !(isfinite(p[0]) && isfinite(p[1]) && isfinite(p[2]) && isfinite(p[3]));
    double x1, y1, x2, y2;
    to_camera(p, K, x1, y1, x2, y2);
    rows32[r] = make_float4((float)x1, (float)y1, (float)x2, (float)y2);
  }
  bad = __syncthreads_or(bad);
  if (tid == 0) {
    for (int j = 0; j < 9; ++j) st->best[j] = 0.0;
    st->n = m;
    st->bad = bad;
    st->stop = bad || m < kSample;
    st->best_count = 0;
    st->K = K;
    st->th2 = ess_th2(px_th, K);
    st->n_all = n;
    st->row0 = pr.row0;
    st->row32 = pr.row0 - B.base;
  }
}

// Hypotheses first .. first + count - 1.  models [count * kSlots][9] fp64 (camera coordinates), counts
// [count * kSlots] (-1: no model in that slot).
__global__ void __launch_bounds__(kScoreThreads, 1) ess_round_kernel(const EssState* __restrict__ st_all,
                                                                  const float4* __restrict__ rows32_all,
                                                                  const double* __restrict__ rows_all, int stride,
                                                                  int first, int count, unsigned long long seed,
                                                                  int ignore_stop, double* __restrict__ models_all,
                                                                  int* __restrict__ counts_all) {
  constexpr int NM = kHypPerBlock * kSlots, NJ = NM / 8;
  __shared__ float4 s_rows[kTile];
  __shared__ double s_M[kHypPerBlock][10][20];
  __shared__ float s_model[NM][9];
  __shared__ int s_valid[NM];
  const EssState* st = st_all + blockIdx.y;
  if (!ignore_stop && st->stop) return;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const int n = st->n;
  const Intrinsics K = st->K;
  const float th2 = st->th2;
  const double* rows = rows_all + st->row0 * stride;
  const float4* rows32 = rows32_all + st->row32;
  double* models = models_all + blockIdx.y * kPairModels;
  int* counts = counts_all + blockIdx.y * kPairCounts;
  if (tid < kHypPerBlock) {
    const int local = blockIdx.x * kHypPerBlock + tid;
    double out[kSlots][9];
    int nm = 0;
    if (local < count) {
      int idx[kSample];
      if (draw_sample<kSample>(seed, first + local, n, idx)) {
        double p[kSample][4];
#pragma unroll
        for (int k = 0; k < kSample; ++k) to_camera(rows + (size_t)idx[k] * stride, K, p[k][0], p[k][1], p[k][2], p[k][3]);
        nm = solve_e5(p, s_M[tid], out);
      }
    }
    for (int k = 0; k < kSlots; ++k) {
      const int slot = tid * kSlots + k;
      s_valid[slot] = k < nm;
      for (int j = 0; j < 9; ++j) {
        s_model[slot][j] = k < nm ? (float)out[k][j] : 0.f;
        if (local < count) models[((size_t)local * kSlots + k) * 9 + j] = k < nm ? out[k][j] : 0.0;
      }
    }
  }
  int cnt[NJ];
#pragma unroll
  for (int j = 0; j < NJ; ++j) cnt[j] = 0;
  for (int t0 = 0; t0 < n; t0 += kTile) {
    const int tn = min(kTile, n - t0);
    __syncthreads();
    for (int r = tid; r < tn; r += kScoreThreads) s_rows[r] = rows32[t0 + r];
    __syncthreads();
#pragma unroll
    for (int j = 0; j < NJ; ++j) {
      const int mi = wid + 8 * j;
      if (!s_valid[mi]) continue;
      float m[9];
#pragma unroll
      for (int e = 0; e < 9; ++e) m[e] = s_model[mi][e];
      for (int r0 = 0; r0 < tn; r0 += 32) {
        const int r = r0 + lane;
        const bool in = r < tn && is_inlier_e(m, s_rows[r < tn ? r : 0], th2);
        cnt[j] += __popc(__ballot_sync(0xffffffffu, in));
      }
    }
  }
  if (lane == 0) {
#pragma unroll
    for (int j = 0; j < NJ; ++j) {
      const int mi = wid + 8 * j;
      const int local = blockIdx.x * kHypPerBlock + mi / kSlots;
      if (local < count) counts[(size_t)blockIdx.x * NM + mi] = s_valid[mi] ? cnt[j] : -1;
    }
  }
}

__global__ void __launch_bounds__(1024) ess_select_kernel(EssState* __restrict__ st, const double* __restrict__ models,
                                                          const int* __restrict__ counts, int nm, int done, double conf,
                                                          int max_iters) {
  select_round(st + blockIdx.y, models + blockIdx.y * kPairModels, counts + blockIdx.y * kPairCounts, nm, done, kSample,
               conf, max_iters);
}

// Local optimisation + outputs: 8-point refit on the inliers (fp64 normal matrix, Jacobi), projected onto the essential
// manifold (singular values 1, 1, 0) at unit Frobenius norm, kept while it has strictly more inliers.
__global__ void __launch_bounds__(kLoThreads, 1) ess_lo_kernel(const EssState* __restrict__ st_all,
                                                            const float4* __restrict__ rows32_all,
                                                            const double* __restrict__ rows_all, int stride,
                                                            double* __restrict__ E_out, uint8_t* __restrict__ mask_out,
                                                            int* __restrict__ count_out) {
  __shared__ double s_red[kLoThreads / 32][45];
  __shared__ double s_cur[9], s_cand[9];
  __shared__ float s_f32[9];
  __shared__ int s_cnt[kLoThreads / 32], s_ok;
  const EssState* st = st_all + blockIdx.y;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const int n = st->n, bad = st->bad, n_all = st->n_all;
  const Intrinsics K = st->K;
  const float th2 = st->th2;
  const double* rows = rows_all + st->row0 * stride;
  const float4* rows32 = rows32_all + st->row32;
  E_out += 9 * blockIdx.y;
  count_out += blockIdx.y;
  mask_out += st->row0;
  int cur_count = bad ? 0 : st->best_count;
  if (tid < 9) s_cur[tid] = st->best[tid];
  __syncthreads();

  auto count_inliers = [&](const double* m64) -> int {    // block-wide, fixed order
    if (tid < 9) s_f32[tid] = (float)m64[tid];
    __syncthreads();
    float m[9];
#pragma unroll
    for (int e = 0; e < 9; ++e) m[e] = s_f32[e];
    int c = 0;
    for (int r = tid; r < n; r += kLoThreads) c += is_inlier_e(m, rows32[r], th2);
    for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
    if (lane == 0) s_cnt[wid] = c;
    __syncthreads();
    int tot = 0;
    for (int w = 0; w < kLoThreads / 32; ++w) tot += s_cnt[w];
    __syncthreads();
    return tot;
  };

  for (int it = 0; it < kLoIters && cur_count >= kLoMin; ++it) {
    if (tid < 9) s_f32[tid] = (float)s_cur[tid];
    __syncthreads();
    float m[9];
#pragma unroll
    for (int e = 0; e < 9; ++e) m[e] = s_f32[e];
    double acc[45];
#pragma unroll
    for (int e = 0; e < 45; ++e) acc[e] = 0.0;
    for (int r = tid; r < n; r += kLoThreads) {
      if (!is_inlier_e(m, rows32[r], th2)) continue;
      double x, y, u, v;
      to_camera(rows + (size_t)r * stride, K, x, y, u, v);
      const double a[9] = {u * x, u * y, u, v * x, v * y, v, x, y, 1.0};
      int e = 0;
#pragma unroll
      for (int i = 0; i < 9; ++i)
#pragma unroll
        for (int j = i; j < 9; ++j) acc[e++] += a[i] * a[j];
    }
#pragma unroll
    for (int e = 0; e < 45; ++e) {
      const double v = warp_sum_d(acc[e]);
      if (lane == 0) s_red[wid][e] = v;
    }
    __syncthreads();
    if (tid == 0) {
      double M[9][9], h[9];
      int e = 0;
      for (int i = 0; i < 9; ++i)
        for (int j = i; j < 9; ++j) {
          double v = 0.0;
          for (int w = 0; w < kLoThreads / 32; ++w) v += s_red[w][e];
          M[i][j] = M[j][i] = v;
          ++e;
        }
      jacobi_min_eigvec<9>(M, h);
      double U[3][3], s[3], Vm[3][3];
      bool ok = svd3(h, U, s, Vm);
      if (ok) {
        double nrm = 0.0;
        for (int i = 0; i < 3; ++i)
          for (int j = 0; j < 3; ++j) {
            const double v = U[i][0] * Vm[j][0] + U[i][1] * Vm[j][1];
            s_cand[3 * i + j] = v;
            nrm += v * v;
          }
        nrm = 1.0 / sqrt(nrm);
        for (int j = 0; j < 9; ++j) s_cand[j] *= nrm;
      }
      s_ok = ok;
    }
    __syncthreads();
    if (!s_ok) break;
    const int c = count_inliers(s_cand);
    if (c <= cur_count) break;
    cur_count = c;
    if (tid < 9) s_cur[tid] = s_cand[tid];
    __syncthreads();
  }

  if (tid < 9) E_out[tid] = bad ? __longlong_as_double(0x7ff8000000000000ll) : (cur_count > 0 ? s_cur[tid] : 0.0);
  if (tid == 0) *count_out = bad ? -1 : cur_count;
  if (tid < 9) s_f32[tid] = (float)s_cur[tid];
  __syncthreads();
  float m[9];
#pragma unroll
  for (int e = 0; e < 9; ++e) m[e] = s_f32[e];
  for (int r = tid; r < n_all; r += kLoThreads) mask_out[r] = cur_count > 0 && r < n && is_inlier_e(m, rows32[r], th2);
}

// ---- pose recovery kernels ----------------------------------------------------------------------------------------
// cv2.decomposeEssentialMat: E = U S V^T with det U, det V^T made positive; R1 = U W V^T, R2 = U W^T V^T, t = U[:, 2].
__global__ void pose_decompose_kernel(PairBatch B, const double* __restrict__ intr, Intrinsics K1,
                                      const double* __restrict__ E, PoseState* __restrict__ ps) {
  if (threadIdx.x != 0) return;
  const int p = blockIdx.y;
  const PairRange pr = pair_range(B, p);
  ps += p;
  E += 9 * (size_t)p;
  ps->K = pair_intrinsics(intr, K1, p);
  ps->n_all = pr.n;
  ps->row0 = pr.row0;
  ps->row32 = pr.row0 - B.base;
  ps->n = effective_rows(pr.n, B.n_dev == nullptr ? nullptr : B.n_dev + p);
  double e[9], amax = 0.0;
  bool fin = true;
  for (int j = 0; j < 9; ++j) {
    e[j] = E[j];
    fin &= isfinite(e[j]);
    amax = fmax(amax, fabs(e[j]));
  }
  double U[3][3], s[3], Vm[3][3];
  const bool ok = fin && amax > 0.0 && svd3(e, U, s, Vm);
  ps->valid = ok;
  if (!ok) return;
  if (det3m(U) < 0.0)
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) U[i][j] = -U[i][j];
  if (det3m(Vm) < 0.0)
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) Vm[i][j] = -Vm[i][j];
  // U W = [-u1, u0, u2], U W^T = [u1, -u0, u2]
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) {
      ps->R[0][3 * i + j] = -U[i][1] * Vm[j][0] + U[i][0] * Vm[j][1] + U[i][2] * Vm[j][2];
      ps->R[1][3 * i + j] = U[i][1] * Vm[j][0] - U[i][0] * Vm[j][1] + U[i][2] * Vm[j][2];
    }
  for (int i = 0; i < 3; ++i) ps->t[i] = U[i][2];
}

// cv2.recoverPose's test of one row against [I|0] and [R|t]: linear triangulation (smallest eigenvector of the 4x4
// normal matrix of the DLT system), then Q2 Q3 > 0, depth in camera 1 below dist_th, depth in camera 2 in (0, dist_th).
__device__ bool good_point(const double* R, const double* t, double x1, double y1, double x2, double y2, double dist_th) {
  const double A[4][4] = {{-1.0, 0.0, x1, 0.0},
                          {0.0, -1.0, y1, 0.0},
                          {x2 * R[6] - R[0], x2 * R[7] - R[1], x2 * R[8] - R[2], x2 * t[2] - t[0]},
                          {y2 * R[6] - R[3], y2 * R[7] - R[4], y2 * R[8] - R[5], y2 * t[2] - t[1]}};
  double N[4][4], q[4];
  for (int i = 0; i < 4; ++i)
    for (int j = 0; j < 4; ++j) N[i][j] = A[0][i] * A[0][j] + A[1][i] * A[1][j] + A[2][i] * A[2][j] + A[3][i] * A[3][j];
  jacobi_min_eigvec<4>(N, q);
  if (!(q[2] * q[3] > 0.0)) return false;
  const double X = q[0] / q[3], Y = q[1] / q[3], Z = q[2] / q[3];
  if (!(Z < dist_th)) return false;
  const double z2 = R[6] * X + R[7] * Y + R[8] * Z + t[2];
  return z2 > 0.0 && z2 < dist_th;
}

__global__ void __launch_bounds__(kPoseThreads) pose_count_kernel(const PoseState* __restrict__ ps,
                                                                  const double* __restrict__ rows, int stride,
                                                                  const uint8_t* __restrict__ mask_in, double dist_th,
                                                                  uint8_t* __restrict__ codes,
                                                                  int* __restrict__ partial) {
  __shared__ int s_cnt[kPoseThreads / 32][4];
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  ps += blockIdx.y;
  const int n = ps->valid ? ps->n : 0;
  const Intrinsics K = ps->K;
  rows += ps->row0 * stride;
  if (mask_in != nullptr) mask_in += ps->row0;
  codes += ps->row32;
  partial += (size_t)blockIdx.y * kPoseBlocks * 4;
  int c[4] = {0, 0, 0, 0};
  for (int r = blockIdx.x * kPoseThreads + tid; r < n; r += kPoseBlocks * kPoseThreads) {
    int code = 0;
    if (mask_in == nullptr || mask_in[r]) {
      double x1, y1, x2, y2;
      to_camera(rows + (size_t)r * stride, K, x1, y1, x2, y2);
      const double tn[3] = {-ps->t[0], -ps->t[1], -ps->t[2]};
#pragma unroll
      for (int k = 0; k < 4; ++k)
        if (good_point(ps->R[k & 1], k < 2 ? ps->t : tn, x1, y1, x2, y2, dist_th)) {
          code |= 1 << k;
          ++c[k];
        }
    }
    codes[r] = (uint8_t)code;
  }
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    int v = c[k];
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (lane == 0) s_cnt[wid][k] = v;
  }
  __syncthreads();
  if (tid < 4) {
    int tot = 0;
    for (int w = 0; w < kPoseThreads / 32; ++w) tot += s_cnt[w][tid];
    partial[blockIdx.x * 4 + tid] = tot;
  }
}

// Candidate with the most good points (ties to the first in OpenCV's order) -> Rt_out [12] (R row-major, t), count,
// mask.  No valid E: zeros and an empty mask.
__global__ void __launch_bounds__(1024) pose_select_kernel(const PoseState* __restrict__ ps,
                                                           const int* __restrict__ partial,
                                                           const uint8_t* __restrict__ codes,
                                                           double* __restrict__ Rt_out, uint8_t* __restrict__ mask_out,
                                                           int* __restrict__ count_out) {
  __shared__ int s_tot[4], s_best;
  const int tid = threadIdx.x;
  ps += blockIdx.y;
  const int valid = ps->valid, n = ps->n, n_all = ps->n_all;
  partial += (size_t)blockIdx.y * kPoseBlocks * 4;
  codes += ps->row32;
  Rt_out += 12 * blockIdx.y;
  count_out += blockIdx.y;
  mask_out += ps->row0;
  if (tid < 4) {
    int tot = 0;
    for (int b = 0; b < kPoseBlocks; ++b) tot += partial[b * 4 + tid];
    s_tot[tid] = tot;
  }
  __syncthreads();
  if (tid == 0) {
    int b = 0;
    for (int k = 1; k < 4; ++k)
      if (s_tot[k] > s_tot[b]) b = k;
    s_best = b;
  }
  __syncthreads();
  const int b = s_best;
  if (tid < 12) {
    const double v = tid < 9 ? ps->R[b & 1][tid] : (b < 2 ? ps->t[tid - 9] : -ps->t[tid - 9]);
    Rt_out[tid] = valid ? v : 0.0;
  }
  if (tid == 0) *count_out = valid ? s_tot[b] : 0;
  for (int r = tid; r < n_all; r += 1024) mask_out[r] = valid && r < n && ((codes[r] >> b) & 1);
}

struct EssScratch {
  EssState* st;
  float4* rows32;
  double* models;
  int* counts;
};

// `pairs` states, `rows` fp32 rows, then nhyp hypotheses' models and counts per pair (nhyp = kRound: pair strides
// kPairModels / kPairCounts).
EssScratch carve_ess(void* base, int pairs, long long rows, int nhyp) {
  char* p = (char*)base;
  EssScratch s;
  s.st = (EssState*)p;
  p += align_up((size_t)pairs * sizeof(EssState), 1024);
  s.rows32 = (float4*)p;
  p += align_up((size_t)rows * sizeof(float4) + 16, 1024);
  s.models = (double*)p;
  p += align_up((size_t)pairs * nhyp * kSlots * 9 * sizeof(double), 1024);
  s.counts = (int*)p;
  return s;
}

}  // namespace

size_t essential_scratch_bytes(int pairs, long long rows, bool rounds) {
  return align_up((size_t)pairs * sizeof(EssState), 1024) + align_up((size_t)rows * sizeof(float4) + 16, 1024) +
         (rounds ? align_up((size_t)pairs * kPairModels * sizeof(double), 1024) + (size_t)pairs * kPairCounts * sizeof(int)
                 : 0);
}

// states, per-block partial counts of every pair, then one code byte per row
size_t pose_scratch_bytes(int pairs, long long rows) {
  return align_up((size_t)pairs * sizeof(PoseState), 1024) + align_up((size_t)pairs * kPoseBlocks * 4 * sizeof(int), 1024) +
         (size_t)rows + 16;
}

int essential_chunk_pairs() {
  const size_t per_pair = sizeof(EssState) + kPairModels * sizeof(double) + kPairCounts * sizeof(int);
  return (int)std::min<size_t>(kMaxGridY, std::max<size_t>(1, kBatchScratchBudget / per_pair));
}

int pose_chunk_pairs() {
  const size_t per_pair = sizeof(PoseState) + kPoseBlocks * 4 * sizeof(int);
  return (int)std::min<size_t>(kMaxGridY, std::max<size_t>(1, kBatchScratchBudget / per_pair));
}

int launch_find_essential(const PairBatch& B, const double* intr, const Intrinsics& K1, double px_th, double conf,
                          int max_iters, unsigned long long seed, void* scratch, double* E_out, uint8_t* mask_out,
                          int* count_out, cudaStream_t st) {
  const EssScratch s = carve_ess(scratch, B.pairs, B.total, kRound);
  const dim3 one(1, B.pairs);
  ess_prep_kernel<<<one, 1024, 0, st>>>(B, intr, K1, px_th, s.rows32, s.st);
  P2P_LAUNCH_OK();
  for (int first = 0; first < max_iters; first += kRound) {
    const int count = min(kRound, max_iters - first);
    ess_round_kernel<<<dim3(cdiv(count, kHypPerBlock), B.pairs), kScoreThreads, 0, st>>>(
        s.st, s.rows32, B.rows, B.stride, first, count, seed, 0, s.models, s.counts);
    P2P_LAUNCH_OK();
    ess_select_kernel<<<one, 1024, 0, st>>>(s.st, s.models, s.counts, count * kSlots, first + count, conf, max_iters);
    P2P_LAUNCH_OK();
  }
  ess_lo_kernel<<<one, kLoThreads, 0, st>>>(s.st, s.rows32, B.rows, B.stride, E_out, mask_out, count_out);
  P2P_LAUNCH_OK();
  return 0;
}

int launch_test_essential_hypotheses(const double* rows, int stride, int n, const Intrinsics& K, double px_th,
                                     unsigned long long seed, int count, void* scratch, double* models_out,
                                     int* counts_out, cudaStream_t st) {
  const PairBatch B = single_pair(rows, stride, n, nullptr);
  const EssScratch s = carve_ess(scratch, 1, n, 0);
  ess_prep_kernel<<<1, 1024, 0, st>>>(B, nullptr, K, px_th, s.rows32, s.st);
  P2P_LAUNCH_OK();
  ess_round_kernel<<<cdiv(count, kHypPerBlock), kScoreThreads, 0, st>>>(s.st, s.rows32, rows, stride, 0, count, seed, 1,
                                                                        models_out, counts_out);
  P2P_LAUNCH_OK();
  return 0;
}

int launch_recover_pose(const PairBatch& B, const double* intr, const Intrinsics& K1, const double* E,
                        const uint8_t* mask_in, double dist_th, void* scratch, double* Rt_out, uint8_t* mask_out,
                        int* count_out, cudaStream_t st) {
  char* p = (char*)scratch;
  PoseState* ps = (PoseState*)p;
  p += align_up((size_t)B.pairs * sizeof(PoseState), 1024);
  int* partial = (int*)p;
  p += align_up((size_t)B.pairs * kPoseBlocks * 4 * sizeof(int), 1024);
  uint8_t* codes = (uint8_t*)p;
  pose_decompose_kernel<<<dim3(1, B.pairs), 32, 0, st>>>(B, intr, K1, E, ps);
  P2P_LAUNCH_OK();
  pose_count_kernel<<<dim3(kPoseBlocks, B.pairs), kPoseThreads, 0, st>>>(ps, B.rows, B.stride, mask_in, dist_th, codes,
                                                                          partial);
  P2P_LAUNCH_OK();
  pose_select_kernel<<<dim3(1, B.pairs), 1024, 0, st>>>(ps, partial, codes, Rt_out, mask_out, count_out);
  P2P_LAUNCH_OK();
  return 0;
}

}  // namespace p2p
