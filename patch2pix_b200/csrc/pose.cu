// Relative pose on the device: RANSAC for an essential matrix (5-point minimal solver) with local optimisation, and
// pose recovery from E (cv2.findEssentialMat(..., RANSAC) + cv2.recoverPose semantics, utils/eval/geometry.py:32-48).
//
// p2p_find_essential runs the RANSAC kernels of verify_common.cuh as kind 3, with no host sync: the prep kernel maps
// the rows to camera coordinates, each round draws 5-point samples -> up to 10 models (one thread each) and scores
// every (model, row) pair in fp32 (Sampson error), and LO refits with the 8-point method projected onto the essential
// manifold.  This file adds what only E needs: the 5-point solver, the projection, and pose recovery.
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
#include "verify_common.cuh"

namespace p2p {
namespace {

constexpr int kMaxRoots = 10;       // real roots of the degree-10 polynomial
constexpr int kBisect = 64;         // bisection steps per root
constexpr int kNewton = 2;          // guarded Newton steps per root
constexpr double kZMax = 1e6;       // roots are searched in (-kZMax, kZMax]
constexpr int kPoseBlocks = 256;
constexpr int kPoseThreads = 256;

struct PoseState {
  double R[2][9], t[3];             // R1, R2 row-major, t = U[:, 2]
  Intrinsics K;                     // the pair's cameras
  int n;                            // effective row count
  int valid;                        // E was finite and non-zero
  int n_all;                        // rows of the pair (mask length)
  long long row0;                   // first row of the pair in the row array and the masks
  long long row32;                  // first row of the pair in the codes
};

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
__device__ int solve_e5(const double (&p)[5][4], double (*M)[20], double (&out)[kMaxRoots][9]) {
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

// ---- E: kind 3 of the RANSAC kernels (verify_common.cuh) ---------------------------------------------------------
// Camera coordinates throughout, scored as F.  kTile = 1024 rows (16 KB) leaves room for the 5-point solver's 12.8 KB
// of shared elimination matrices: 2048 would put the round kernel 384 bytes under the 48 KB static shared-memory limit.
template <> struct Kind<3> : TwoView<3> {
  static constexpr int kSample = 5, kSlots = kMaxRoots, kPairSlots = kMaxRoots, kLoMin = 8, kScore = 0, kTile = 1024;
  // Thread t < kHypPerBlock of a round block solves its hypothesis with s_M[t] as its elimination matrix.
  static __device__ int solve(const VerifyState&, const double (&p)[5][4], double (&out)[kSlots][9]) {
    __shared__ double s_M[kHypPerBlock][10][20];
    return solve_e5(p, s_M[threadIdx.x], out);
  }
  // The refit projected onto the essential manifold (singular values 1, 1, 0) at unit Frobenius norm.
  static __device__ bool refit(const VerifyState&, double (&h)[9], double* out) {
    double U[3][3], s[3], Vm[3][3];
    if (!svd3(h, U, s, Vm)) return false;
    double nrm = 0.0;
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) {
        const double v = U[i][0] * Vm[j][0] + U[i][1] * Vm[j][1];
        out[3 * i + j] = v;
        nrm += v * v;
      }
    nrm = 1.0 / sqrt(nrm);
    for (int j = 0; j < 9; ++j) out[j] *= nrm;
    return true;
  }
};

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
  ps->n = effective_rows(B, p, pr.n);
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

}  // namespace

size_t essential_scratch_bytes(int pairs, long long rows, bool rounds) { return scratch_bytes<3>(pairs, rows, rounds); }

// states, per-block partial counts of every pair, then one code byte per row
size_t pose_scratch_bytes(int pairs, long long rows) {
  return align_up((size_t)pairs * sizeof(PoseState), 1024) + align_up((size_t)pairs * kPoseBlocks * 4 * sizeof(int), 1024) +
         (size_t)rows + 16;
}

int essential_chunk_pairs() { return chunk_pairs<3>(); }

int pose_chunk_pairs() {
  const size_t per_pair = sizeof(PoseState) + kPoseBlocks * 4 * sizeof(int);
  return (int)std::min<size_t>(kMaxGridY, std::max<size_t>(1, kBatchScratchBudget / per_pair));
}

int launch_find_essential(const PairBatch& B, const double* intr, const Intrinsics& K1, double px_th,
                          const double* px_th_dev, double conf, int max_iters, unsigned long long seed, void* scratch,
                          double* E_out, uint8_t* mask_out, int* count_out, cudaStream_t st) {
  return find_model<3>(B, intr, K1, px_th, px_th_dev, conf, max_iters, seed, scratch, E_out, mask_out, count_out, st);
}

int launch_test_essential_hypotheses(const double* rows, int stride, int n, const Intrinsics& K, double px_th,
                                     unsigned long long seed, int count, void* scratch, double* models_out,
                                     int* counts_out, cudaStream_t st) {
  return test_hypotheses<3>(rows, stride, n, K, px_th, seed, count, scratch, models_out, counts_out, st);
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
