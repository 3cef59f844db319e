// Device helpers of the RANSAC engine (verify_common.cuh), pose recovery (pose.cu) and the epipolar histograms
// (eval.cu): a batch's row ranges, the counter-based sample generator, fp64 null space and smallest-eigenvector
// solvers, the Sampson terms, fixed-order block sums and the per-round select / stop rule.  Everything here is inlined
// into the calling kernels of each translation unit.
#pragma once
#include <math.h>

#include "kernels.h"

namespace p2p {
namespace {

constexpr int kMaxDraws = 64;       // draws per sample before it counts as degenerate

// Rows of pair p of a batch: rows offsets[p] .. offsets[p+1]-1 of the row array, or all n1 rows of a single pair.
struct PairRange {
  long long row0;
  int n;
};
__device__ __forceinline__ PairRange pair_range(const PairBatch& B, int p) {
  if (B.offsets == nullptr) return PairRange{0, B.n1};
  const long long r0 = B.offsets[p];
  return PairRange{r0, (int)(B.offsets[p + 1] - r0)};
}
// Rows pair p uses of its n: n_dev[p] when that lies in [0, n), else n.
__device__ __forceinline__ int effective_rows(const PairBatch& B, int p, int n) {
  if (B.n_dev != nullptr) {
    const double v = B.n_dev[p];
    if (v >= 0.0 && v < (double)n) return (int)v;
  }
  return n;
}

// ---- stateless sample generator: index `draw` of hypothesis `hyp` (restated in oracle/verify_oracle.py) -------------
__device__ __forceinline__ unsigned long long mix64(unsigned long long z) {   // splitmix64 finaliser
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}
__device__ __forceinline__ int draw_index(unsigned long long seed, int hyp, int draw, int n) {
  const unsigned long long key = seed * 0xD1B54A32D192ED03ull +
                                 ((unsigned long long)hyp * kMaxDraws + (unsigned long long)draw) * 0x9E3779B97F4A7C15ull +
                                 0x632BE59BD9B4E019ull;
  return (int)(((mix64(key) >> 32) * (unsigned long long)n) >> 32);
}
// S distinct row indices; a repeated index is re-drawn.  False after kMaxDraws draws.
template <int S>
__device__ bool draw_sample(unsigned long long seed, int hyp, int n, int (&idx)[S]) {
  int d = 0;
#pragma unroll
  for (int k = 0; k < S; ++k) {
    bool dup = true;
    while (dup) {
      if (d >= kMaxDraws) return false;
      idx[k] = draw_index(seed, hyp, d++, n);
      dup = false;
#pragma unroll
      for (int j = 0; j < k; ++j) dup |= idx[j] == idx[k];
    }
  }
  return true;
}

// ---- fp64 linear algebra (one thread) ----------------------------------------------------------------------------
// Null space of the R x 9 system A by full-pivoting Gauss-Jordan elimination: ns[f] has a 1 in the f-th free column.
// False when A is rank deficient (a pivot below 1e-9 of the largest entry).
template <int R>
__device__ bool null_space(double (&A)[R][9], double (&ns)[9 - R][9]) {
  int perm[9];
  double amax0 = 0.0;
  for (int j = 0; j < 9; ++j) perm[j] = j;
  for (int i = 0; i < R; ++i)
    for (int j = 0; j < 9; ++j) amax0 = fmax(amax0, fabs(A[i][j]));
  if (!(amax0 > 0.0)) return false;
  for (int k = 0; k < R; ++k) {
    int p = k, q = k;
    double best = -1.0;
    for (int i = k; i < R; ++i)
      for (int j = k; j < 9; ++j)
        if (fabs(A[i][j]) > best) { best = fabs(A[i][j]); p = i; q = j; }
    if (!(best > 1e-9 * amax0)) return false;
    for (int j = 0; j < 9; ++j) { const double t = A[k][j]; A[k][j] = A[p][j]; A[p][j] = t; }
    for (int i = 0; i < R; ++i) { const double t = A[i][k]; A[i][k] = A[i][q]; A[i][q] = t; }
    { const int t = perm[k]; perm[k] = perm[q]; perm[q] = t; }
    const double piv = A[k][k];
    for (int j = 0; j < 9; ++j) A[k][j] /= piv;
    for (int i = 0; i < R; ++i) {
      if (i == k) continue;
      const double f = A[i][k];
      for (int j = 0; j < 9; ++j) A[i][j] -= f * A[k][j];
    }
  }
  for (int f = 0; f < 9 - R; ++f) {
    for (int j = 0; j < 9; ++j) ns[f][j] = 0.0;
    ns[f][perm[R + f]] = 1.0;
    for (int i = 0; i < R; ++i) ns[f][perm[i]] = -A[i][R + f];
  }
  return true;
}

// Eigenvector of the smallest eigenvalue of the symmetric N x N matrix M (destroyed), cyclic Jacobi.
template <int N>
__device__ void jacobi_min_eigvec(double (&M)[N][N], double (&v)[N]) {
  double V[N][N];
  for (int i = 0; i < N; ++i)
    for (int j = 0; j < N; ++j) V[i][j] = i == j ? 1.0 : 0.0;
  for (int sweep = 0; sweep < 50; ++sweep) {
    double off = 0.0, diag = 0.0;
    for (int p = 0; p < N; ++p) {
      diag += M[p][p] * M[p][p];
      for (int q = p + 1; q < N; ++q) off += M[p][q] * M[p][q];
    }
    if (!(off > 1e-30 * diag)) break;
    for (int p = 0; p < N - 1; ++p)
      for (int q = p + 1; q < N; ++q) {
        const double apq = M[p][q];
        if (apq == 0.0) continue;
        const double theta = (M[q][q] - M[p][p]) / (2.0 * apq);
        const double t = fabs(theta) > 1e150 ? 0.5 / theta : copysign(1.0, theta) / (fabs(theta) + sqrt(theta * theta + 1.0));
        const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
        for (int k = 0; k < N; ++k) {
          const double mkp = M[k][p], mkq = M[k][q];
          M[k][p] = c * mkp - s * mkq;
          M[k][q] = s * mkp + c * mkq;
        }
        for (int k = 0; k < N; ++k) {
          const double mpk = M[p][k], mqk = M[q][k];
          M[p][k] = c * mpk - s * mqk;
          M[q][k] = s * mpk + c * mqk;
        }
        for (int k = 0; k < N; ++k) {
          const double vkp = V[k][p], vkq = V[k][q];
          V[k][p] = c * vkp - s * vkq;
          V[k][q] = s * vkp + c * vkq;
        }
      }
  }
  int jm = 0;
  for (int j = 1; j < N; ++j)
    if (M[j][j] < M[jm][jm]) jm = j;
  for (int i = 0; i < N; ++i) v[i] = V[i][jm];
}

// ---- scoring ------------------------------------------------------------------------------------------------------
// Sampson terms of the reference's sampson_distance (measure.py:36-39): dd = x2^T F x1 and the squared norms of the
// first two coordinates of l2 = F x1 and l1 = F^T x2.
template <typename T>
__device__ __forceinline__ void sampson_terms(const T* m, T x1, T y1, T x2, T y2, T& dd, T& den) {
  const T l2x = m[0] * x1 + m[1] * y1 + m[2], l2y = m[3] * x1 + m[4] * y1 + m[5], l2z = m[6] * x1 + m[7] * y1 + m[8];
  const T l1x = m[0] * x2 + m[3] * y2 + m[6], l1y = m[1] * x2 + m[4] * y2 + m[7];
  dd = x2 * l2x + y2 * l2y + l2z;
  den = l1x * l1x + l1y * l1y + l2x * l2x + l2y * l2y;
}

// The reference's sampson_distance of one row (measure.py:36-39, eps = 1e-8): the one expression of both
// p2p_sampson_distance (verify.cu) and p2p_epipolar_histograms (eval.cu).
__device__ __forceinline__ double sampson_distance(const double* m, const double* p) {
  double dd, den;
  sampson_terms<double>(m, p[0], p[1], p[2], p[3], dd, den);
  return dd * dd / (1e-8 + den);
}

__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__device__ __forceinline__ double block_sum_1024(double v, double* red) {   // fixed-order sum over 1024 threads
  v = warp_sum_d(v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  v = threadIdx.x < 32 ? red[threadIdx.x] : 0.0;
  if (threadIdx.x < 32) v = warp_sum_d(v);
  if (threadIdx.x == 0) red[32] = v;
  __syncthreads();
  return red[32];
}

// ---- per-round selection (one block of 1024 threads) --------------------------------------------------------------
// Best of this round's nm models -> state if strictly better than the best so far (most inliers, ties to the lowest
// (hypothesis, root) index); then the stopping bound log(1-conf) / log(1-w^s).  State has best[L], n, stop, best_count;
// models holds L doubles per model (9 for F / H / E, 12 for an absolute pose).  `past_stop` selects even when an earlier
// select of the same round has set stop (extra candidates of that round).
template <int L = 9, typename State>
__device__ __forceinline__ void select_round(State* __restrict__ st, const double* __restrict__ models,
                                             const int* __restrict__ counts, int nm, int done, int sample, double conf,
                                             int max_iters, bool past_stop = false) {
  __shared__ unsigned long long red[32];
  if (st->stop && !past_stop) return;
  const int tid = threadIdx.x;
  unsigned long long key = 0;     // (count, lowest index first)
  for (int m = tid; m < nm; m += 1024) {
    const int c = counts[m];
    const unsigned long long k = c > 0 ? ((unsigned long long)c << 32) | (0xFFFFFFFFull - (unsigned)m) : 0ull;
    key = k > key ? k : key;
  }
  for (int o = 16; o > 0; o >>= 1) {
    const unsigned long long x = __shfl_xor_sync(0xffffffffu, key, o);
    key = x > key ? x : key;
  }
  if ((tid & 31) == 0) red[tid >> 5] = key;
  __syncthreads();
  if (tid >= 32) return;
  key = red[tid];
  for (int o = 16; o > 0; o >>= 1) {
    const unsigned long long x = __shfl_xor_sync(0xffffffffu, key, o);
    key = x > key ? x : key;
  }
  if (tid != 0) return;
  const int c = (int)(key >> 32);
  if (c > st->best_count) {
    const int m = (int)(0xFFFFFFFFull - (key & 0xFFFFFFFFull));
    st->best_count = c;
    for (int j = 0; j < L; ++j) st->best[j] = models[(size_t)m * L + j];
  }
  double needed = HUGE_VAL;
  if (st->best_count > 0) {
    const double ws = pow((double)st->best_count / (double)st->n, (double)sample);
    needed = ws >= 1.0 ? 0.0 : log(1.0 - conf) / log1p(-ws);
  }
  st->stop = done >= max_iters || (double)done >= needed;
}

}  // namespace
}  // namespace p2p
