// DEGENSAC (Chum, Werner & Matas, CVPR 2005) on the device: F RANSAC (model 2 of p2p_find_model) with the plane-
// degeneracy test and plane-and-parallax rounds.  Per round of model 0's launches (verify_common.cuh) it adds:
//   verify_degen_kernel    (1 block)  before the select: H-degeneracy test of the round's records (the slots a
//                                     sequential RANSAC would adopt); the first degenerate one sets `pending` and its
//                                     induced H
// and, after the select, three launches that return at once unless `pending` is set:
//   verify_plane_kernel    (1 block)  DLT refit of that H on the rows within h_th while the count grows (fp64)
//   verify_round_kernel<2> (x1 round) kRound plane-and-parallax models F = [e']x H, scored as F
//   verify_parallax_select_kernel      adopts the best of them if it has strictly more inliers, clears `pending`
// A batch of pairs adds grid dimension y to each launch, one block per pair (verify_common.cuh).
// Testing every record rather than only the round's winner matters: a round of 1024 hypotheses often ends RANSAC on a
// dominant-plane scene, and its winner is frequently a sample with 4 coplanar points, or with 5 whose induced H is
// too noisy to pass the test, while an earlier record is degenerate.
#include <limits.h>
#include <math.h>

#include "kernels.h"
#include "verify_common.cuh"

namespace p2p {
namespace {

// ---- DEGENSAC ------------------------------------------------------------------------------------------------------
__constant__ int kTriplets[5][3] = {{0, 1, 2}, {3, 4, 5}, {0, 1, 6}, {3, 4, 6}, {2, 5, 6}};

// H-degeneracy test of the 7-point sample of hypothesis `hyp` under its pixel model F (one thread, fp64).  In Hartley-
// normalised coordinates, for each triplet in kTriplets: e' the unit left null vector of F (the largest cross product
// of two columns), A = [e']x F, M the rows x_i^T, b_i = (x'_i x A x_i)^T (x'_i x e') / |x'_i x e'|^2 and the induced
// H = A - e' (M^-1 b)^T (Hartley & Zisserman, result 13.6).  The sample is degenerate when at least kDegenMin of its 7
// points lie within h_th of H (h_inlier64, pixels).  Returns the first degenerate triplet (its pixel H in H_out) or -1;
// a vanishing e', a point at the epipole or collinear x_i give that triplet no H.
__device__ int degeneracy_test(const VerifyState& S, const double* F, int hyp, const double* rows, int stride,
                               unsigned long long seed, double h_th2, double* H_out) {
  int idx[7];
  if (!draw_sample<7>(seed, hyp, S.n, idx)) return -1;
  double Fn[9], tmp[9];
  {
    const double T2it[9] = {1.0 / S.s[1], 0.0, 0.0, 0.0, 1.0 / S.s[1], 0.0, S.cx[1], S.cy[1], 1.0};
    const double T1i[9] = {1.0 / S.s[0], 0.0, S.cx[0], 0.0, 1.0 / S.s[0], S.cy[0], 0.0, 0.0, 1.0};
    mat3_mul(T2it, F, tmp);
    mat3_mul(tmp, T1i, Fn);
  }
  double e[3], fn2 = 0.0, en = -1.0;
  for (int j = 0; j < 9; ++j) fn2 += Fn[j] * Fn[j];
  {
    const double c[3][3] = {{Fn[0], Fn[3], Fn[6]}, {Fn[1], Fn[4], Fn[7]}, {Fn[2], Fn[5], Fn[8]}};
    const int pr[3][2] = {{0, 1}, {0, 2}, {1, 2}};
    for (int k = 0; k < 3; ++k) {
      double x[3];
      cross3(c[pr[k][0]], c[pr[k][1]], x);
      const double nx = sqrt(dot3(x, x));
      if (nx > en) { en = nx; e[0] = x[0]; e[1] = x[1]; e[2] = x[2]; }
    }
  }
  if (!(en > 1e-10 * fn2)) return -1;
  for (int k = 0; k < 3; ++k) e[k] /= en;
  double A[9];
  skew_mul(e, Fn, A);
  for (int t = 0; t < 5; ++t) {
    double M[9], b[3];
    bool ok = true;
    for (int i = 0; i < 3 && ok; ++i) {
      const double* r = rows + (size_t)idx[kTriplets[t][i]] * stride;
      const double x1[3] = {(r[0] - S.cx[0]) * S.s[0], (r[1] - S.cy[0]) * S.s[0], 1.0};
      const double x2[3] = {(r[2] - S.cx[1]) * S.s[1], (r[3] - S.cy[1]) * S.s[1], 1.0};
      M[3 * i] = x1[0]; M[3 * i + 1] = x1[1]; M[3 * i + 2] = 1.0;
      double c[3], ax[3], q[3];
      cross3(x2, e, c);
      const double cc = dot3(c, c);
      ok = cc > 1e-12 * dot3(x2, x2);
      for (int j = 0; j < 3; ++j) ax[j] = A[3 * j] * x1[0] + A[3 * j + 1] * x1[1] + A[3 * j + 2];
      cross3(x2, ax, q);
      b[i] = dot3(q, c) / cc;
    }
    if (!ok) continue;
    const double det = det3(M);
    double rn = 1.0;
    for (int i = 0; i < 3; ++i) rn *= sqrt(M[3 * i] * M[3 * i] + M[3 * i + 1] * M[3 * i + 1] + 1.0);
    if (!(fabs(det) > 1e-10 * rn)) continue;
    const double inv[9] = {M[4] * M[8] - M[5] * M[7], M[2] * M[7] - M[1] * M[8], M[1] * M[5] - M[2] * M[4],
                           M[5] * M[6] - M[3] * M[8], M[0] * M[8] - M[2] * M[6], M[2] * M[3] - M[0] * M[5],
                           M[3] * M[7] - M[4] * M[6], M[1] * M[6] - M[0] * M[7], M[0] * M[4] - M[1] * M[3]};
    double v[3];
    for (int j = 0; j < 3; ++j) v[j] = (inv[3 * j] * b[0] + inv[3 * j + 1] * b[1] + inv[3 * j + 2] * b[2]) / det;
    double Hn[9];
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) Hn[3 * i + j] = A[3 * i + j] - e[i] * v[j];
    if (!denormalise<1>(S, Hn, tmp)) continue;
    int c = 0;
    for (int k = 0; k < 7; ++k) c += h_inlier64(tmp, rows + (size_t)idx[k] * stride, h_th2);
    if (c >= kDegenMin) {
      for (int j = 0; j < 9; ++j) H_out[j] = tmp[j];
      return t;
    }
  }
  return -1;
}

// DEGENSAC, before the select of an F round: the round's records -- slots whose count beats the best so far and every
// earlier slot of the round, i.e. the models a sequential RANSAC would adopt -- are tested in slot order; the first
// degenerate one sets `pending` and its induced H (st->plane).  Slots are scanned in contiguous chunks per thread with
// a fixed-order exclusive max-scan, so the result does not depend on scheduling.
__global__ void __launch_bounds__(kDegenThreads, 1) verify_degen_kernel(VerifyState* __restrict__ st_all,
                                                                     const double* __restrict__ models_all,
                                                                     const int* __restrict__ counts_all, int nm, int first,
                                                                     const double* __restrict__ rows_all, int stride,
                                                                     unsigned long long seed, double h_th2) {
  constexpr int kChunk = kRound * 3 / kDegenThreads;
  __shared__ int s_max[kDegenThreads / 32], s_first[kDegenThreads / 32];
  VerifyState* st = st_all + blockIdx.y;
  if (st->stop) return;
  const double* models = models_all + blockIdx.y * kPairModels<0>;
  const int* counts = counts_all + blockIdx.y * kPairCounts<0>;
  const double* rows = rows_all + st->row0 * stride;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5, m0 = tid * kChunk;
  int mx = 0;
  for (int k = 0; k < kChunk && m0 + k < nm; ++k) mx = max(mx, counts[m0 + k]);
  int inc = mx;                                               // inclusive max-scan over the block
  for (int o = 1; o < 32; o <<= 1) {
    const int y = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc = max(inc, y);
  }
  if (lane == 31) s_max[wid] = inc;
  __syncthreads();
  int run = max(st->best_count, __shfl_up_sync(0xffffffffu, inc, 1) * (lane > 0));
  for (int w = 0; w < wid; ++w) run = max(run, s_max[w]);
  int found = INT_MAX;
  double H[9];
  for (int k = 0; k < kChunk && m0 + k < nm; ++k) {
    const int c = counts[m0 + k];
    if (c <= run) continue;
    run = c;
    if (found == INT_MAX &&
        degeneracy_test(*st, models + (size_t)(m0 + k) * 9, first + (m0 + k) / 3, rows, stride, seed, h_th2, H) >= 0)
      found = m0 + k;
  }
  int f = found;                                              // first degenerate record of the block
  for (int o = 16; o > 0; o >>= 1) f = min(f, __shfl_xor_sync(0xffffffffu, f, o));
  if (lane == 0) s_first[wid] = f;
  __syncthreads();
  f = INT_MAX;
  for (int w = 0; w < kDegenThreads / 32; ++w) f = min(f, s_first[w]);
  if (found != INT_MAX && found == f)
    for (int j = 0; j < 9; ++j) st->plane[j] = H[j];
  if (tid == 0) st->pending = f != INT_MAX;
}

// DEGENSAC: the plane of a pending round -- DLT refit of st->plane on the rows within h_th (fp64 tests, normalised
// coordinates), kept while the count grows, as the H path of verify_lo_kernel.
__global__ void __launch_bounds__(kLoThreads, 1) verify_plane_kernel(VerifyState* __restrict__ st_all,
                                                                  const double* __restrict__ rows_all, int stride,
                                                                  double h_th2) {
  __shared__ double s_red[kLoThreads / 32][45];
  __shared__ double s_cur[9], s_cand[9];
  __shared__ int s_cnt[kLoThreads / 32], s_ok;
  VerifyState* st = st_all + blockIdx.y;
  if (!st->pending) return;
  const double* rows = rows_all + st->row0 * stride;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const int n = st->n;
  if (tid < 9) s_cur[tid] = st->plane[tid];
  __syncthreads();
  auto count_inliers = [&](const double* H) -> int {      // block-wide, fixed order
    int c = 0;
    for (int r = tid; r < n; r += kLoThreads) c += h_inlier64(H, rows + (size_t)r * stride, h_th2);
    for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
    if (lane == 0) s_cnt[wid] = c;
    __syncthreads();
    int tot = 0;
    for (int w = 0; w < kLoThreads / 32; ++w) tot += s_cnt[w];
    __syncthreads();
    return tot;
  };
  int cur_count = count_inliers(s_cur);
  for (int it = 0; it < kLoIters && cur_count >= Kind<1>::kLoMin; ++it) {
    double acc[45];
#pragma unroll
    for (int e = 0; e < 45; ++e) acc[e] = 0.0;
    const double c1x = st->cx[0], c1y = st->cy[0], s1 = st->s[0], c2x = st->cx[1], c2y = st->cy[1], s2 = st->s[1];
    for (int r = tid; r < n; r += kLoThreads) {
      const double* p = rows + (size_t)r * stride;
      if (!h_inlier64(s_cur, p, h_th2)) continue;
      const double x = (p[0] - c1x) * s1, y = (p[1] - c1y) * s1, u = (p[2] - c2x) * s2, v = (p[3] - c2y) * s2;
      const double a[9] = {-x, -y, -1.0, 0.0, 0.0, 0.0, u * x, u * y, u};
      const double b[9] = {0.0, 0.0, 0.0, -x, -y, -1.0, v * x, v * y, v};
      int e = 0;
#pragma unroll
      for (int i = 0; i < 9; ++i)
#pragma unroll
        for (int j = i; j < 9; ++j) acc[e++] += a[i] * a[j] + b[i] * b[j];
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
      s_ok = denormalise<1>(*st, h, s_cand);
    }
    __syncthreads();
    if (!s_ok) break;
    const int c = count_inliers(s_cand);
    if (c <= cur_count) break;
    cur_count = c;
    if (tid < 9) s_cur[tid] = s_cand[tid];
    __syncthreads();
  }
  if (tid < 9) st->plane[tid] = s_cur[tid];
}

// DEGENSAC: best plane-and-parallax model of a pending round -> state if strictly better, stopping bound as for F;
// then the round is done.
__global__ void __launch_bounds__(1024) verify_parallax_select_kernel(VerifyState* __restrict__ st,
                                                                      const double* __restrict__ models,
                                                                      const int* __restrict__ counts, int done,
                                                                      double conf, int max_iters) {
  st += blockIdx.y;
  if (!st->pending) return;
  select_round(st, models + blockIdx.y * kPairModels<0>, counts + blockIdx.y * kPairCounts<0>, kRound, done,
               Kind<0>::kSample, conf, max_iters, true);
  if (threadIdx.x == 0) st->pending = 0;
}

// Test hook: the degeneracy test of every slot of hypotheses 0 .. count-1 (models / counts of verify_round_kernel<0>).
__global__ void verify_degen_hook_kernel(const VerifyState* __restrict__ st, const double* __restrict__ models,
                                         const int* __restrict__ counts, int nslots, const double* __restrict__ rows,
                                         int stride, unsigned long long seed, double h_th2, int* __restrict__ tri_out,
                                         double* __restrict__ H_out) {
  const int m = blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= nslots) return;
  double H[9] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
  int t = -2;
  if (counts[m] >= 0) t = degeneracy_test(*st, models + (size_t)m * 9, m / 3, rows, stride, seed, h_th2, H);
  tri_out[m] = t;
  for (int j = 0; j < 9; ++j) H_out[(size_t)m * 9 + j] = t >= 0 ? H[j] : 0.0;
}

// DEGENSAC (model 2): model 0's rounds, select and LO, plus the degeneracy test and plane-and-parallax launches of
// every round; h_th = 2 px_th.
int find_model_degensac(const PairBatch& B, double px_th, double conf, int max_iters, unsigned long long seed,
                        void* scratch, double* model_out, uint8_t* mask_out, int* count_out, cudaStream_t st) {
  const Scratch s = carve<0>(scratch, B.pairs, B.total, kRound);
  const double h_th2 = (2.0 * px_th) * (2.0 * px_th);
  const dim3 one(1, B.pairs);
  verify_prep_kernel<false><<<one, 1024, 0, st>>>(B, nullptr, {}, px_th, nullptr, Kind<0>::kSample, s.rows32, s.st);
  P2P_LAUNCH_OK();
  for (int first = 0; first < max_iters; first += kRound) {
    const int count = min(kRound, max_iters - first);
    int rc = enqueue_round<0>(s, B, first, count, seed, 0, st);
    if (rc) return rc;
    verify_degen_kernel<<<one, kDegenThreads, 0, st>>>(s.st, s.models, s.counts, count * 3, first, B.rows, B.stride, seed,
                                                       h_th2);
    P2P_LAUNCH_OK();
    verify_select_kernel<<<one, 1024, 0, st>>>(s.st, s.models, s.counts, count * 3, first + count, Kind<0>::kSample,
                                               Kind<0>::kPairSlots, conf, max_iters);
    P2P_LAUNCH_OK();
    verify_plane_kernel<<<one, kLoThreads, 0, st>>>(s.st, B.rows, B.stride, h_th2);
    P2P_LAUNCH_OK();
    if ((rc = enqueue_round<2>(s, B, first, kRound, seed, 0, st, h_th2))) return rc;
    verify_parallax_select_kernel<<<one, 1024, 0, st>>>(s.st, s.models, s.counts, first + count, conf, max_iters);
    P2P_LAUNCH_OK();
  }
  verify_lo_kernel<0><<<one, kLoThreads, 0, st>>>(s.st, s.rows32, B.rows, B.stride, model_out, mask_out, count_out);
  P2P_LAUNCH_OK();
  return 0;
}

}  // namespace

size_t verify_degeneracy_scratch_bytes(int n, int count) {
  return verify_scratch_bytes(1, n, false) + align_up((size_t)count * 3 * 9 * sizeof(double), 1024) +
         (size_t)count * 3 * sizeof(int);
}

int launch_test_degeneracy(const double* rows, int stride, int n, double px_th, unsigned long long seed, int count,
                           void* scratch, int* tri_out, double* H_out, cudaStream_t st) {
  const PairBatch B = single_pair(rows, stride, n, nullptr);
  Scratch s = carve<0>(scratch, 1, n, count);
  const double h_th2 = (2.0 * px_th) * (2.0 * px_th);
  verify_prep_kernel<false><<<1, 1024, 0, st>>>(B, nullptr, {}, px_th, nullptr, Kind<0>::kSample, s.rows32, s.st);
  P2P_LAUNCH_OK();
  int rc = enqueue_round<0>(s, B, 0, count, seed, 1, st);
  if (rc) return rc;
  verify_degen_hook_kernel<<<cdiv(count * 3, 128), 128, 0, st>>>(s.st, s.models, s.counts, count * 3, rows, stride, seed,
                                                                 h_th2, tri_out, H_out);
  P2P_LAUNCH_OK();
  return 0;
}

int launch_find_model_degensac(const PairBatch& B, double px_th, double conf, int max_iters, unsigned long long seed,
                               void* scratch, double* model_out, uint8_t* mask_out, int* count_out, cudaStream_t st) {
  return find_model_degensac(B, px_th, conf, max_iters, seed, scratch, model_out, mask_out, count_out, st);
}

}  // namespace p2p
