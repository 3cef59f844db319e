// Triangulation of a detector-free matcher's matches against known poses, and query 2D-3D rows for localization.
//
// Every stage is deterministic: ids come from radix-sorted keys (CUB's sort is stable), never from atomic counters, and
// every floating-point sum runs in a fixed order in one thread.  This file is compiled with -fmad=false, so each
// product and sum is rounded on its own and oracle/sfm_oracle.py, written in the same order, reproduces the keypoint
// means, the undistortion and the query rows bit for bit.
//
//   keypoints   endpoint keys (image << 44 | cell_y << 22 | cell_x) -> stable sort -> one keypoint per key, id = rank,
//               position = mean of its endpoints in input order (one thread sums a key's run of the sorted array)
//   undistort   fixed-iteration Newton inverse of COLMAP's radial distortion, one thread per keypoint
//   tracks      first-in-pair rule by two stable sorts of (pair, keypoint) keys, Sampson test under the model's E,
//               unique edges by a sort, connected components by atomicMin hooking + pointer jumping until no hook
//               changes a label (one host sync), observations sorted by (label, keypoint)
//   triangulate one block per track: hypotheses spread over the threads, the best by a shared atomicMax of
//               (score + 1) << 32 | ~index, refinement, acceptance and bookkeeping in thread 0 in observation order
//   query rows  query keypoints by the keypoint stage; each database endpoint's nearest triangulated keypoint in the
//               3x3 cells around it (binary search of the sorted keys); unique (query keypoint, point) keys by a sort
#include <cub/cub.cuh>

#include "common.cuh"
#include "kernels.h"

namespace p2p {
namespace {

constexpr int kSfmThreads = 256;
constexpr int kTriThreads = 128;
constexpr int kTriSample = 32;               // hypotheses: pairs among the first 32 remaining observations
constexpr int kUndistortIters = 12;
constexpr int kGaussNewtonSteps = 5;
constexpr int kMaxTrackObs = 1 << 16;
constexpr unsigned long long kNoKey = ~0ull;
constexpr double kCells = 4194304.0;         // 2^22 cells per axis

inline unsigned grid_of(long long n) { return (unsigned)((n + kSfmThreads - 1) / kSfmThreads); }

// Largest p in [0, P) with offsets[p] <= m (offsets[0] = 0, offsets[P] = M > m): the pair of match m.
__device__ __forceinline__ int pair_of(const long long* offsets, int P, long long m) {
  int lo = 0, hi = P;
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (offsets[mid] <= m) lo = mid;
    else hi = mid;
  }
  return lo;
}

__device__ __forceinline__ long long ep_match(long long e, int both) { return both ? e >> 1 : e; }
__device__ __forceinline__ int ep_side(long long e, int both) { return both ? (int)(e & 1) : 0; }

__device__ __forceinline__ unsigned long long cell_key(long long img, double x, double y, double px) {
  if (!(isfinite(x) && isfinite(y) && x >= 0.0 && y >= 0.0)) return kNoKey;
  const double cx = floor(x / px), cy = floor(y / px);
  if (!(cx < kCells && cy < kCells)) return kNoKey;
  return ((unsigned long long)img << 44) | ((unsigned long long)cy << 22) | (unsigned long long)cx;
}

// ---- keypoints ------------------------------------------------------------------------------------------------------
__global__ void ep_key_kernel(const double* __restrict__ m4, long long M, const long long* __restrict__ offsets, int P,
                              const int* __restrict__ pair_img, int both, double px, unsigned long long* keys,
                              int* vals, long long* counts) {
  const long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (e >= (both ? 2 * M : M)) return;
  const long long m = ep_match(e, both);
  const int s = ep_side(e, both);
  const int p = pair_of(offsets, P, m);
  const unsigned long long k = cell_key(pair_img[2 * p + s], m4[4 * m + 2 * s], m4[4 * m + 2 * s + 1], px);
  if (k == kNoKey) atomicAdd((unsigned long long*)&counts[1], 1ull);
  keys[e] = k;
  vals[e] = (int)e;
}

// flag[i] = 1 where a run of equal valid keys starts
__global__ void head_flag_kernel(const unsigned long long* __restrict__ keys, long long n, int* flag) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= n) return;
  const unsigned long long k = keys[i];
  flag[i] = k != kNoKey && (i == 0 || keys[i - 1] != k);
}

__global__ void kp_mean_kernel(const unsigned long long* __restrict__ keys, const int* __restrict__ vals,
                               const int* __restrict__ ids, long long E, const double* __restrict__ m4, int both,
                               double* kp_xy, unsigned long long* kp_key, int* kp_of_ep, long long* counts) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= E) return;
  const unsigned long long k = keys[i];
  kp_of_ep[vals[i]] = k == kNoKey ? -1 : ids[i] - 1;
  if (i == E - 1) counts[0] = ids[i];
  if (k == kNoKey || (i > 0 && keys[i - 1] == k)) return;
  double sx = 0.0, sy = 0.0;
  long long c = 0;
  for (long long j = i; j < E && keys[j] == k; ++j, ++c) {
    const long long e = vals[j], m = ep_match(e, both);
    const int s = ep_side(e, both);
    sx = sx + m4[4 * m + 2 * s];
    sy = sy + m4[4 * m + 2 * s + 1];
  }
  const int id = ids[i] - 1;
  kp_xy[2 * id] = sx / (double)c;
  kp_xy[2 * id + 1] = sy / (double)c;
  kp_key[id] = k;
}

// ---- cameras: record [8] = model, fx, fy, cx, cy, k1, k2, 0 (k2 = 0 for SIMPLE_RADIAL, k1 = k2 = 0 for pinholes) ------
__device__ void undistort(const double* c, double xd, double yd, double& u, double& v) {
  const double x = (xd - c[3]) / c[1], y = (yd - c[4]) / c[2], k1 = c[5], k2 = c[6];
  u = x;
  v = y;
  for (int it = 0; it < kUndistortIters; ++it) {
    const double u2 = u * u, v2 = v * v, uv = u * v, r2 = u2 + v2;
    const double rad = k1 * r2 + k2 * r2 * r2, dr = k1 + 2.0 * k2 * r2;
    const double fu = u + u * rad - x, fv = v + v * rad - y;
    const double a = 1.0 + rad + 2.0 * u2 * dr, b = 2.0 * uv * dr, d = 1.0 + rad + 2.0 * v2 * dr;
    const double det = a * d - b * b;
    u = u - (d * fu - b * fv) / det;
    v = v - (a * fv - b * fu) / det;
  }
}

__device__ __forceinline__ void distort_px(const double* c, double u, double v, double& px, double& py) {
  const double r2 = u * u + v * v, rad = c[5] * r2 + c[6] * r2 * r2;
  px = c[1] * (u + u * rad) + c[3];
  py = c[2] * (v + v * rad) + c[4];
}

__global__ void undistort_kernel(const double* __restrict__ xy, const unsigned long long* __restrict__ key,
                                 long long cap, const long long* __restrict__ n_dev, const int* __restrict__ img_cam,
                                 const double* __restrict__ cams, double* out) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= cap || (n_dev != nullptr && i >= *n_dev)) return;
  const double* c = cams + 8 * (size_t)img_cam[key[i] >> 44];
  undistort(c, xy[2 * i], xy[2 * i + 1], out[2 * i], out[2 * i + 1]);
}

// ---- tracks ---------------------------------------------------------------------------------------------------------
__global__ void side_key_kernel(const int* __restrict__ kp_of_ep, long long M, const long long* __restrict__ offsets,
                                int P, int side, unsigned long long* keys, int* vals) {
  const long long m = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (m >= M) return;
  const int k = kp_of_ep[2 * m + side];
  keys[m] = k < 0 ? kNoKey : ((unsigned long long)pair_of(offsets, P, m) << 32) | (unsigned)k;
  vals[m] = (int)m;
}

__global__ void first_flag_kernel(const unsigned long long* __restrict__ keys, const int* __restrict__ vals,
                                  long long n, unsigned char* first) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= n) return;
  const unsigned long long k = keys[i];
  if (k != kNoKey && (i == 0 || keys[i - 1] != k)) first[vals[i]] = 1;
}

__global__ void edge_key_kernel(const int* __restrict__ kp_of_ep, long long M, const long long* __restrict__ offsets,
                                int P, const unsigned char* __restrict__ firstA,
                                const unsigned char* __restrict__ firstB, const double* __restrict__ E,
                                const double* __restrict__ thr, const double* __restrict__ kp_n,
                                unsigned long long* keys, long long* counts) {
  const long long m = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (m >= M) return;
  unsigned long long key = kNoKey;
  if (firstA[m] && firstB[m]) {
    const int ka = kp_of_ep[2 * m], kb = kp_of_ep[2 * m + 1];
    const int p = pair_of(offsets, P, m);
    const double* e = E + 9 * (size_t)p;
    const double a0 = kp_n[2 * ka], a1 = kp_n[2 * ka + 1], b0 = kp_n[2 * kb], b1 = kp_n[2 * kb + 1];
    const double e0 = e[0] * a0 + e[1] * a1 + e[2], e1 = e[3] * a0 + e[4] * a1 + e[5], e2 = e[6] * a0 + e[7] * a1 + e[8];
    const double f0 = e[0] * b0 + e[3] * b1 + e[6], f1 = e[1] * b0 + e[4] * b1 + e[7];
    const double num = b0 * e0 + b1 * e1 + e2;
    const double s = num * num / (e0 * e0 + e1 * e1 + f0 * f0 + f1 * f1);
    atomicAdd((unsigned long long*)&counts[4], 1ull);
    if (s <= thr[p] && ka != kb)
      key = ka < kb ? ((unsigned long long)ka << 32) | (unsigned)kb : ((unsigned long long)kb << 32) | (unsigned)ka;
  }
  keys[m] = key;
}

// state[0]: a hook changed a label in this iteration; state[1]: converged (later iterations return at once)
__global__ void hook_kernel(const unsigned long long* __restrict__ edges, long long n, int* label, int* state,
                            long long* counts, int first) {
  if (state[1]) return;
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= n) return;
  const unsigned long long k = edges[i];
  if (k == kNoKey || (i > 0 && edges[i - 1] == k)) return;
  if (first) atomicAdd((unsigned long long*)&counts[0], 1ull);
  const int lu = label[(int)(k >> 32)], lv = label[(int)(k & 0xffffffffu)];
  if (lu != lv) {
    atomicMin(&label[max(lu, lv)], min(lu, lv));
    state[0] = 1;
  }
}

__global__ void jump_kernel(int* label, long long n, const int* state) {
  if (state[1]) return;
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= n) return;
  int l = label[i];
  for (int nx = ((volatile int*)label)[l]; nx != l; nx = ((volatile int*)label)[l]) l = nx;
  label[i] = l;
}

__global__ void converge_kernel(int* state) {
  if (state[1]) return;
  if (state[0] == 0) state[1] = 1;
  state[0] = 0;
}

__global__ void iota_kernel(int* v, long long n) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i < n) v[i] = (int)i;
}

// flag[i] = 1 where a track of 2 .. 2^16 observations starts; len[i] its length there
__global__ void track_flag_kernel(const int* __restrict__ lab, long long n, int* flag, int* len, long long* counts) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= n) return;
  flag[i] = 0;
  if (i > 0 && lab[i - 1] == lab[i]) return;
  long long j = i + 1;
  while (j < n && lab[j] == lab[i]) ++j;
  const long long l = j - i;
  len[i] = (int)min(l, (long long)INT_MAX);
  if (l > kMaxTrackObs) atomicAdd((unsigned long long*)&counts[3], 1ull);
  else if (l >= 2) {
    flag[i] = 1;
    atomicAdd((unsigned long long*)&counts[2], (unsigned long long)l);
  }
}

__global__ void track_table_kernel(const int* __restrict__ flag, const int* __restrict__ ids,
                                   const int* __restrict__ len, long long n, int* start, int* tlen, long long* counts) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= n) return;
  if (i == n - 1) counts[1] = ids[i];
  if (!flag[i]) return;
  start[ids[i] - 1] = (int)i;
  tlen[ids[i] - 1] = len[i];
}

// ---- triangulation --------------------------------------------------------------------------------------------------
// image record [15]: R row-major, t, centre C = -R^T t
struct TriArgs {
  const int *obs_kp, *start, *len;
  const double *kp_xy, *kp_n;
  const unsigned long long* kp_key;
  const double* img;
  const int* img_cam;
  const double* cams;
  double th2, cos_min;
  double* slot_X;        // [tracks * kMaxSfmTrackPoints][3]
  int* slot_len;         // 0: no point
  double* slot_err;
  int* obs_slot;         // sorted-observation index -> slot, -1 (none) ; -2 while remaining
};

__device__ __forceinline__ int obs_image(const TriArgs& a, int o) { return (int)(a.kp_key[a.obs_kp[o]] >> 44); }

// squared reprojection error of observation o in original pixels, or -1 when the depth is not positive
__device__ double reproj_err2(const TriArgs& a, int o, const double* X) {
  const int im = obs_image(a, o);
  const double* r = a.img + 15 * (size_t)im;
  const double p0 = r[0] * X[0] + r[1] * X[1] + r[2] * X[2] + r[9];
  const double p1 = r[3] * X[0] + r[4] * X[1] + r[5] * X[2] + r[10];
  const double p2 = r[6] * X[0] + r[7] * X[1] + r[8] * X[2] + r[11];
  if (!(p2 > 0.0)) return -1.0;
  double px, py;
  distort_px(a.cams + 8 * (size_t)a.img_cam[im], p0 / p2, p1 / p2, px, py);
  const int k = a.obs_kp[o];
  const double dx = px - a.kp_xy[2 * k], dy = py - a.kp_xy[2 * k + 1];
  return dx * dx + dy * dy;
}

__device__ __forceinline__ bool is_inlier(const TriArgs& a, int o, const double* X) {
  const double e = reproj_err2(a, o, X);
  return e >= 0.0 && e <= a.th2;
}

// number of distinct images with an inlier among the remaining observations (observations of an image are adjacent)
__device__ int score_point(const TriArgs& a, int o0, int n, const double* X) {
  int score = 0, cur = -1;
  bool counted = false;
  for (int o = o0; o < o0 + n; ++o) {
    if (a.obs_slot[o] != -2) continue;
    const int im = obs_image(a, o);
    if (im != cur) {
      cur = im;
      counted = false;
    }
    if (!counted && is_inlier(a, o, X)) {
      ++score;
      counted = true;
    }
  }
  return score;
}

// 3x3 symmetric solve by the adjugate: M = [m00 m01 m02; . m11 m12; . . m22]
__device__ bool solve3(const double* m, const double* b, double* x) {
  const double c00 = m[4] * m[8] - m[5] * m[5], c01 = m[2] * m[5] - m[1] * m[8], c02 = m[1] * m[5] - m[2] * m[4];
  const double c11 = m[0] * m[8] - m[2] * m[2], c12 = m[1] * m[2] - m[0] * m[5], c22 = m[0] * m[4] - m[1] * m[1];
  const double det = m[0] * c00 + m[1] * c01 + m[2] * c02;
  if (!(det != 0.0) || !isfinite(det)) return false;
  x[0] = (c00 * b[0] + c01 * b[1] + c02 * b[2]) / det;
  x[1] = (c01 * b[0] + c11 * b[1] + c12 * b[2]) / det;
  x[2] = (c02 * b[0] + c12 * b[1] + c22 * b[2]) / det;
  return isfinite(x[0]) && isfinite(x[1]) && isfinite(x[2]);
}

// accumulate the two DLT rows x P2 - P0, y P2 - P1 of a normalised observation into A^T A (m, 9) and A^T b (v, 3)
__device__ void dlt_rows(const double* r, double x, double y, double* m, double* v) {
  for (int q = 0; q < 2; ++q) {
    const double s = q == 0 ? x : y;
    const double a0 = s * r[6] - r[3 * q], a1 = s * r[7] - r[3 * q + 1], a2 = s * r[8] - r[3 * q + 2];
    const double b = r[9 + q] - s * r[11];
    m[0] = m[0] + a0 * a0; m[1] = m[1] + a0 * a1; m[2] = m[2] + a0 * a2;
    m[4] = m[4] + a1 * a1; m[5] = m[5] + a1 * a2; m[8] = m[8] + a2 * a2;
    v[0] = v[0] + a0 * b; v[1] = v[1] + a1 * b; v[2] = v[2] + a2 * b;
  }
}

// two-view linear triangulation of observations i, j; valid iff both depths are positive and the angle >= min_angle
__device__ bool two_view(const TriArgs& a, int oi, int oj, double* X) {
  double m[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0}, v[3] = {0, 0, 0};
  const int ii = obs_image(a, oi), ij = obs_image(a, oj);
  const int ki = a.obs_kp[oi], kj = a.obs_kp[oj];
  dlt_rows(a.img + 15 * (size_t)ii, a.kp_n[2 * ki], a.kp_n[2 * ki + 1], m, v);
  dlt_rows(a.img + 15 * (size_t)ij, a.kp_n[2 * kj], a.kp_n[2 * kj + 1], m, v);
  m[3] = m[1]; m[6] = m[2]; m[7] = m[5];
  if (!solve3(m, v, X)) return false;
  double d[2][3];
  for (int q = 0; q < 2; ++q) {
    const double* r = a.img + 15 * (size_t)(q == 0 ? ii : ij);
    if (!(r[6] * X[0] + r[7] * X[1] + r[8] * X[2] + r[11] > 0.0)) return false;
    for (int c = 0; c < 3; ++c) d[q][c] = X[c] - r[12 + c];
  }
  const double dot = d[0][0] * d[1][0] + d[0][1] * d[1][1] + d[0][2] * d[1][2];
  const double n0 = d[0][0] * d[0][0] + d[0][1] * d[0][1] + d[0][2] * d[0][2];
  const double n1 = d[1][0] * d[1][0] + d[1][1] * d[1][1] + d[1][2] * d[1][2];
  return dot / sqrt(n0 * n1) <= a.cos_min;
}

__device__ bool wide_angle(const TriArgs& a, int ia, int ib, const double* X) {
  const double *ra = a.img + 15 * (size_t)ia, *rb = a.img + 15 * (size_t)ib;
  const double d0[3] = {X[0] - ra[12], X[1] - ra[13], X[2] - ra[14]}, d1[3] = {X[0] - rb[12], X[1] - rb[13], X[2] - rb[14]};
  const double dot = d0[0] * d1[0] + d0[1] * d1[1] + d0[2] * d1[2];
  const double n0 = d0[0] * d0[0] + d0[1] * d0[1] + d0[2] * d0[2], n1 = d1[0] * d1[0] + d1[1] * d1[1] + d1[2] * d1[2];
  return dot / sqrt(n0 * n1) <= a.cos_min;
}

// Gauss-Newton on X over the selected observations (sel[o] = 1), residuals in the normalised plane, fixed order
__device__ void refine_point(const TriArgs& a, int o0, int n, const unsigned char* sel, double* X) {
  for (int step = 0; step < kGaussNewtonSteps; ++step) {
    double m[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0}, g[3] = {0, 0, 0};
    for (int o = o0; o < o0 + n; ++o) {
      if (!sel[o]) continue;
      const double* r = a.img + 15 * (size_t)obs_image(a, o);
      const int k = a.obs_kp[o];
      const double p0 = r[0] * X[0] + r[1] * X[1] + r[2] * X[2] + r[9];
      const double p1 = r[3] * X[0] + r[4] * X[1] + r[5] * X[2] + r[10];
      const double p2 = r[6] * X[0] + r[7] * X[1] + r[8] * X[2] + r[11];
      if (!(p2 > 0.0)) continue;
      const double u = p0 / p2, v = p1 / p2;
      const double ru = u - a.kp_n[2 * k], rv = v - a.kp_n[2 * k + 1];
      double J[2][3];
      for (int c = 0; c < 3; ++c) {
        J[0][c] = (r[c] - u * r[6 + c]) / p2;
        J[1][c] = (r[3 + c] - v * r[6 + c]) / p2;
      }
      for (int q = 0; q < 2; ++q) {
        const double rq = q == 0 ? ru : rv;
        m[0] = m[0] + J[q][0] * J[q][0]; m[1] = m[1] + J[q][0] * J[q][1]; m[2] = m[2] + J[q][0] * J[q][2];
        m[4] = m[4] + J[q][1] * J[q][1]; m[5] = m[5] + J[q][1] * J[q][2]; m[8] = m[8] + J[q][2] * J[q][2];
        g[0] = g[0] - J[q][0] * rq; g[1] = g[1] - J[q][1] * rq; g[2] = g[2] - J[q][2] * rq;
      }
    }
    m[3] = m[1]; m[6] = m[2]; m[7] = m[5];
    double d[3];
    if (!solve3(m, g, d)) return;
    for (int c = 0; c < 3; ++c) X[c] = X[c] + d[c];
  }
}

__global__ void __launch_bounds__(kTriThreads) triangulate_kernel(TriArgs a, unsigned char* sel) {
  __shared__ int s_idx[kTriSample];
  __shared__ int s_n, s_stop;
  __shared__ unsigned long long s_best;
  const int t = blockIdx.x, tid = threadIdx.x;
  const int o0 = a.start[t], n = a.len[t];
  for (int o = o0 + tid; o < o0 + n; o += kTriThreads) {
    a.obs_slot[o] = -2;
    sel[o] = 0;
  }
  __syncthreads();
  int points = 0;
  for (int round = 0; round < kMaxSfmTrackPoints; ++round) {
    if (tid == 0) {
      int cnt = 0, images = 0, cur = -1;
      for (int o = o0; o < o0 + n; ++o) {
        if (a.obs_slot[o] != -2) continue;
        if (cnt < kTriSample) s_idx[cnt++] = o;
        const int im = obs_image(a, o);
        if (im != cur) {
          cur = im;
          ++images;
        }
      }
      s_n = cnt;
      s_stop = images < 2;
      s_best = 0;
    }
    __syncthreads();
    if (s_stop) break;
    const int ns = s_n;
    for (int hyp = tid; hyp < kTriSample * kTriSample; hyp += kTriThreads) {
      const int i = hyp / kTriSample, j = hyp % kTriSample;
      if (j <= i || j >= ns || obs_image(a, s_idx[i]) == obs_image(a, s_idx[j])) continue;
      double X[3];
      if (!two_view(a, s_idx[i], s_idx[j], X)) continue;
      const unsigned long long key =
          ((unsigned long long)(score_point(a, o0, n, X) + 1) << 32) | (0xffffffffu - (unsigned)hyp);
      atomicMax(&s_best, key);
    }
    __syncthreads();
    if (s_best == 0) break;                       // no valid hypothesis
    if (tid == 0) {
      const int hyp = (int)(0xffffffffu - (unsigned)(s_best & 0xffffffffu));
      const int oi = s_idx[hyp / kTriSample], oj = s_idx[hyp % kTriSample];
      const int score = (int)(s_best >> 32) - 1;
      double X[3], Y[3];
      two_view(a, oi, oj, X);
      // one inlier per image: the smallest error, ties to the lower observation
      int cur = -1, best = -1;
      double best_e = 0.0;
      for (int o = o0; o <= o0 + n; ++o) {
        const int im = o < o0 + n ? obs_image(a, o) : -1;
        if (im != cur) {
          if (best >= 0) sel[best] = 1;
          cur = im;
          best = -1;
        }
        if (o == o0 + n || a.obs_slot[o] != -2) continue;
        const double e = reproj_err2(a, o, X);
        if (e >= 0.0 && e <= a.th2 && (best < 0 || e < best_e)) {
          best = o;
          best_e = e;
        }
      }
      for (int c = 0; c < 3; ++c) Y[c] = X[c];
      refine_point(a, o0, n, sel, Y);
      if (score_point(a, o0, n, Y) >= score)
        for (int c = 0; c < 3; ++c) X[c] = Y[c];
      for (int o = o0; o < o0 + n; ++o) sel[o] = 0;
      // inliers of the final point; one representative per image for the angle test
      int images = 0, inl = 0;
      double err = 0.0;
      bool wide = false;
      cur = -1;
      for (int o = o0; o < o0 + n; ++o) {
        if (a.obs_slot[o] != -2) continue;
        const double e = reproj_err2(a, o, X);
        if (!(e >= 0.0 && e <= a.th2)) continue;
        sel[o] = 1;
        ++inl;
        err = err + sqrt(e);
        const int im = obs_image(a, o);
        if (im != cur) {
          cur = im;
          ++images;
          sel[o] = 2;
        }
      }
      for (int p = o0; p < o0 + n && !wide; ++p) {
        if (sel[p] != 2) continue;
        for (int q = p + 1; q < o0 + n && !wide; ++q)
          if (sel[q] == 2) wide = wide_angle(a, obs_image(a, p), obs_image(a, q), X);
      }
      const bool accept = images >= 2 && wide;
      const int slot = t * kMaxSfmTrackPoints + points;
      for (int o = o0; o < o0 + n; ++o) {
        if (sel[o]) a.obs_slot[o] = accept ? slot : -1;
        sel[o] = 0;
      }
      if (a.obs_slot[oi] == -2) a.obs_slot[oi] = -1;
      if (a.obs_slot[oj] == -2) a.obs_slot[oj] = -1;
      if (accept) {
        for (int c = 0; c < 3; ++c) a.slot_X[3 * (size_t)slot + c] = X[c];
        a.slot_len[slot] = inl;
        a.slot_err[slot] = err / (double)inl;
      }
      s_n = accept;
    }
    __syncthreads();
    points += s_n;
    __syncthreads();
  }
  __syncthreads();
  for (int o = o0 + tid; o < o0 + n; o += kTriThreads)
    if (a.obs_slot[o] == -2) a.obs_slot[o] = -1;
}

__global__ void nonzero_flag_kernel(const int* __restrict__ v, long long n, int* flag) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i < n) flag[i] = v[i] != 0;
}

__global__ void point_compact_kernel(const int* __restrict__ slot_len, const int* __restrict__ ids,
                                     const double* __restrict__ slot_X, const double* __restrict__ slot_err,
                                     long long slots, double* pts, int* pt_len, double* pt_err, long long* counts) {
  const long long s = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (s >= slots) return;
  if (s == slots - 1) counts[0] = ids[s];
  if (slot_len[s] == 0) return;
  const int p = ids[s] - 1;
  for (int c = 0; c < 3; ++c) pts[3 * (size_t)p + c] = slot_X[3 * s + c];
  pt_len[p] = slot_len[s];
  pt_err[p] = slot_err[s];
}

__global__ void kp_point_kernel(const int* __restrict__ obs_slot, const int* __restrict__ obs_kp,
                                const int* __restrict__ ids, long long n, int* kp_point) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int s = obs_slot[i];
  kp_point[obs_kp[i]] = s >= 0 ? ids[s] - 1 : -1;
}

// ---- query rows -----------------------------------------------------------------------------------------------------
__device__ long long find_key(const unsigned long long* keys, long long n, unsigned long long k) {
  long long lo = 0, hi = n;
  while (lo < hi) {
    const long long mid = (lo + hi) >> 1;
    if (keys[mid] < k) lo = mid + 1;
    else hi = mid;
  }
  return lo < n && keys[lo] == k ? lo : -1;
}

__global__ void query_key_kernel(const double* __restrict__ m4, long long M, const long long* __restrict__ offsets,
                                 int P, const int* __restrict__ pair_img, double px, const int* __restrict__ qkp_of_ep,
                                 const unsigned long long* __restrict__ kp_key, const double* __restrict__ kp_xy,
                                 const int* __restrict__ kp_point, long long n_kp, unsigned long long* keys) {
  const long long m = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (m >= M) return;
  keys[m] = kNoKey;
  const int q = qkp_of_ep[m];
  const double x = m4[4 * m + 2], y = m4[4 * m + 3];
  const unsigned long long c = cell_key(pair_img[2 * pair_of(offsets, P, m) + 1], x, y, px);
  if (q < 0 || c == kNoKey) return;
  const long long cx = (long long)(c & 0x3fffff), cy = (long long)((c >> 22) & 0x3fffff);
  const unsigned long long img = c >> 44;
  long long best = -1;
  double best_d = 0.0;
  for (long long dy = -1; dy <= 1; ++dy)
    for (long long dx = -1; dx <= 1; ++dx) {
      const long long ny = cy + dy, nx = cx + dx;
      if (ny < 0 || nx < 0 || ny >= (1 << 22) || nx >= (1 << 22)) continue;
      const long long k = find_key(kp_key, n_kp, (img << 44) | ((unsigned long long)ny << 22) | (unsigned long long)nx);
      if (k < 0 || kp_point[k] < 0) continue;
      const double ex = kp_xy[2 * k] - x, ey = kp_xy[2 * k + 1] - y, d = ex * ex + ey * ey;
      if (d <= px * px && (best < 0 || d < best_d || (d == best_d && k < best))) {
        best = k;
        best_d = d;
      }
    }
  if (best >= 0) keys[m] = ((unsigned long long)q << 32) | (unsigned)kp_point[best];
}

__global__ void query_row_kernel(const unsigned long long* __restrict__ keys, const int* __restrict__ ids, long long n,
                                 const unsigned long long* __restrict__ qkp_key, const double* __restrict__ qkp_n,
                                 const double* __restrict__ q_intr, const double* __restrict__ pts, double* rows,
                                 int* q_count) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= n) return;
  const unsigned long long k = keys[i];
  if (k == kNoKey || (i > 0 && keys[i - 1] == k)) return;
  const int qk = (int)(k >> 32), p = (int)(k & 0xffffffffu), r = ids[i] - 1;
  const int q = (int)(qkp_key[qk] >> 44);
  const double* c = q_intr + 4 * (size_t)q;
  rows[5 * (size_t)r] = c[0] * qkp_n[2 * qk] + c[2];
  rows[5 * (size_t)r + 1] = c[1] * qkp_n[2 * qk + 1] + c[3];
  for (int j = 0; j < 3; ++j) rows[5 * (size_t)r + 2 + j] = pts[3 * (size_t)p + j];
  atomicAdd(&q_count[q + 1], 1);
}

__global__ void offsets_kernel(const int* __restrict__ incl, int Q, long long* offsets) {
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q <= Q) offsets[q] = incl[q];
}

// ---- host helpers ---------------------------------------------------------------------------------------------------
size_t sort_bytes(long long n, bool pairs) {
  size_t b = 0;
  if (pairs)
    cub::DeviceRadixSort::SortPairs(nullptr, b, (unsigned long long*)nullptr, (unsigned long long*)nullptr,
                                    (int*)nullptr, (int*)nullptr, (int)n);
  else
    cub::DeviceRadixSort::SortKeys(nullptr, b, (unsigned long long*)nullptr, (unsigned long long*)nullptr, (int)n);
  return b;
}

size_t scan_bytes(long long n) {
  size_t b = 0;
  cub::DeviceScan::InclusiveSum(nullptr, b, (int*)nullptr, (int*)nullptr, (int)n);
  return b;
}

}  // namespace

int launch_sfm_keypoints(Arena& ar, const double* m4, long long M, const long long* offsets, int P,
                         const int* pair_img, int both, double px, double* kp_xy, unsigned long long* kp_key,
                         int* kp_of_ep, long long* counts, cudaStream_t st) {
  const long long E = both ? 2 * M : M;
  const size_t tmp = std::max(sort_bytes(E, true), scan_bytes(E));
  int rc = ar.reserve(4 * align_up(E * 8 + 16, 256) + align_up(tmp + 16, 256) + 4096);
  if (rc) return rc;
  Carve c{(char*)ar.take(ar.cap - 1024)};
  auto* k0 = c.take<unsigned long long>(E);
  auto* k1 = c.take<unsigned long long>(E);
  int* v0 = c.take<int>(E);
  int* v1 = c.take<int>(E);
  int* ids = c.take<int>(E);
  void* t = c.take<char>(tmp);
  P2P_CUDA_OK(cudaMemsetAsync(counts, 0, 2 * sizeof(long long), st));
  if (E == 0) return 0;
  ep_key_kernel<<<grid_of(E), kSfmThreads, 0, st>>>(m4, M, offsets, P, pair_img, both, px, k0, v0, counts);
  P2P_LAUNCH_OK();
  size_t tb = tmp;
  P2P_CUDA_OK(cub::DeviceRadixSort::SortPairs(t, tb, k0, k1, v0, v1, (int)E, 0, 64, st));
  head_flag_kernel<<<grid_of(E), kSfmThreads, 0, st>>>(k1, E, ids);
  P2P_LAUNCH_OK();
  tb = tmp;
  P2P_CUDA_OK(cub::DeviceScan::InclusiveSum(t, tb, ids, ids, (int)E, st));
  kp_mean_kernel<<<grid_of(E), kSfmThreads, 0, st>>>(k1, v1, ids, E, m4, both, kp_xy, kp_key, kp_of_ep, counts);
  P2P_LAUNCH_OK();
  return 0;
}

int launch_sfm_undistort(const double* xy, const unsigned long long* key, long long cap, const long long* n_dev,
                         const int* img_cam, const double* cams, double* out, cudaStream_t st) {
  if (cap == 0) return 0;
  undistort_kernel<<<grid_of(cap), kSfmThreads, 0, st>>>(xy, key, cap, n_dev, img_cam, cams, out);
  P2P_LAUNCH_OK();
  return 0;
}

int launch_sfm_tracks(Arena& ar, const int* kp_of_ep, long long M, const long long* offsets, int P, const double* E,
                      const double* thr, const double* kp_n, long long n_kp, int* labels, int* obs_kp, int* start,
                      int* tlen, long long* counts_dev, long long* counts_host, cudaStream_t st) {
  const long long n = std::max(M, n_kp);
  const size_t tmp = std::max(sort_bytes(n, true), scan_bytes(n));
  int rc = ar.reserve(6 * align_up(n * 8 + 16, 256) + align_up(tmp + 16, 256) + 4096);
  if (rc) return rc;
  Carve c{(char*)ar.take(ar.cap - 1024)};
  auto* k0 = c.take<unsigned long long>(n);
  auto* k1 = c.take<unsigned long long>(n);
  int* v0 = c.take<int>(n);
  int* v1 = c.take<int>(n);
  auto* first = c.take<unsigned char>(2 * n);
  int* flag = c.take<int>(n);
  int* state = c.take<int>(2);
  void* t = c.take<char>(tmp);
  P2P_CUDA_OK(cudaMemsetAsync(counts_dev, 0, 6 * sizeof(long long), st));
  P2P_CUDA_OK(cudaMemsetAsync(first, 0, 2 * n, st));
  P2P_CUDA_OK(cudaMemsetAsync(state, 0, 2 * sizeof(int), st));
  size_t tb;
  for (int side = 0; side < 2 && M > 0; ++side) {
    side_key_kernel<<<grid_of(M), kSfmThreads, 0, st>>>(kp_of_ep, M, offsets, P, side, k0, v0);
    P2P_LAUNCH_OK();
    tb = tmp;
    P2P_CUDA_OK(cub::DeviceRadixSort::SortPairs(t, tb, k0, k1, v0, v1, (int)M, 0, 64, st));
    first_flag_kernel<<<grid_of(M), kSfmThreads, 0, st>>>(k1, v1, M, first + side * n);
    P2P_LAUNCH_OK();
  }
  if (n_kp > 0) {
    iota_kernel<<<grid_of(n_kp), kSfmThreads, 0, st>>>(labels, n_kp);
    P2P_LAUNCH_OK();
  }
  // without keypoints every endpoint was dropped: no match is an edge (and the jump kernel would have no blocks)
  if (M > 0 && n_kp > 0) {
    edge_key_kernel<<<grid_of(M), kSfmThreads, 0, st>>>(kp_of_ep, M, offsets, P, first, first + n, E, thr, kp_n, k0,
                                                        counts_dev);
    P2P_LAUNCH_OK();
    tb = tmp;
    P2P_CUDA_OK(cub::DeviceRadixSort::SortKeys(t, tb, k0, k1, (int)M, 0, 64, st));
    // hooking until no label changes: 16 iterations per host check (components of the edge lists met so far converge in
    // well under 16; the check is the stage's one sync)
    int it = 0;
    for (;;) {
      for (int r = 0; r < 16; ++r, ++it) {
        hook_kernel<<<grid_of(M), kSfmThreads, 0, st>>>(k1, M, labels, state, counts_dev, it == 0);
        P2P_LAUNCH_OK();
        jump_kernel<<<grid_of(n_kp), kSfmThreads, 0, st>>>(labels, n_kp, state);
        P2P_LAUNCH_OK();
        converge_kernel<<<1, 1, 0, st>>>(state);
        P2P_LAUNCH_OK();
      }
      int h_state[2];
      P2P_CUDA_OK(cudaMemcpyAsync(h_state, state, sizeof(h_state), cudaMemcpyDeviceToHost, st));
      P2P_CUDA_OK(cudaStreamSynchronize(st));
      if (h_state[1]) break;
    }
  }
  if (n_kp > 0) {
    iota_kernel<<<grid_of(n_kp), kSfmThreads, 0, st>>>(v0, n_kp);
    P2P_LAUNCH_OK();
    tb = tmp;
    int bits = 1;
    while (bits < 32 && (1ll << bits) < n_kp) ++bits;
    P2P_CUDA_OK(cub::DeviceRadixSort::SortPairs(t, tb, (const unsigned*)labels, (unsigned*)k0, v0, obs_kp, (int)n_kp, 0,
                                                bits, st));
    const int* lab = (const int*)k0;
    track_flag_kernel<<<grid_of(n_kp), kSfmThreads, 0, st>>>(lab, n_kp, flag, v1, counts_dev);
    P2P_LAUNCH_OK();
    tb = tmp;
    P2P_CUDA_OK(cub::DeviceScan::InclusiveSum(t, tb, flag, v0, (int)n_kp, st));
    track_table_kernel<<<grid_of(n_kp), kSfmThreads, 0, st>>>(flag, v0, v1, n_kp, start, tlen, counts_dev);
    P2P_LAUNCH_OK();
  }
  P2P_CUDA_OK(cudaMemcpyAsync(counts_host, counts_dev, 6 * sizeof(long long), cudaMemcpyDeviceToHost, st));
  P2P_CUDA_OK(cudaStreamSynchronize(st));
  return 0;
}

int launch_sfm_triangulate(Arena& ar, const int* obs_kp, const int* start, const int* tlen, int n_tracks,
                           long long n_kp, const double* kp_xy, const double* kp_n, const unsigned long long* kp_key,
                           const double* img, const int* img_cam, const double* cams, double reproj_px,
                           double cos_min, double* pts, int* pt_len, double* pt_err, int* kp_point, long long* counts,
                           cudaStream_t st) {
  const long long slots = (long long)n_tracks * kMaxSfmTrackPoints;
  const size_t tmp = scan_bytes(std::max(slots, 1ll));
  int rc = ar.reserve(align_up(slots * 24 + 16, 256) + 3 * align_up(slots * 8 + 16, 256) +
                      2 * align_up(n_kp * 4 + 16, 256) + align_up(tmp + 16, 256) + 4096);
  if (rc) return rc;
  Carve c{(char*)ar.take(ar.cap - 1024)};
  double* sX = c.take<double>(3 * slots);
  int* slen = c.take<int>(slots);
  double* serr = c.take<double>(slots);
  int* ids = c.take<int>(slots);
  int* obs_slot = c.take<int>(n_kp);
  auto* sel = c.take<unsigned char>(n_kp);
  void* t = c.take<char>(tmp);
  P2P_CUDA_OK(cudaMemsetAsync(counts, 0, sizeof(long long), st));
  if (n_kp > 0) {
    P2P_CUDA_OK(cudaMemsetAsync(obs_slot, 0xff, n_kp * sizeof(int), st));
    P2P_CUDA_OK(cudaMemsetAsync(kp_point, 0xff, n_kp * sizeof(int), st));
  }
  if (n_tracks == 0) return 0;
  P2P_CUDA_OK(cudaMemsetAsync(slen, 0, slots * sizeof(int), st));
  TriArgs a{obs_kp, start, tlen, kp_xy, kp_n, kp_key, img, img_cam, cams, reproj_px * reproj_px, cos_min,
            sX, slen, serr, obs_slot};
  triangulate_kernel<<<n_tracks, kTriThreads, 0, st>>>(a, sel);
  P2P_LAUNCH_OK();
  nonzero_flag_kernel<<<grid_of(slots), kSfmThreads, 0, st>>>(slen, slots, ids);
  P2P_LAUNCH_OK();
  size_t tb = tmp;
  P2P_CUDA_OK(cub::DeviceScan::InclusiveSum(t, tb, ids, ids, (int)slots, st));
  point_compact_kernel<<<grid_of(slots), kSfmThreads, 0, st>>>(slen, ids, sX, serr, slots, pts, pt_len, pt_err, counts);
  P2P_LAUNCH_OK();
  kp_point_kernel<<<grid_of(n_kp), kSfmThreads, 0, st>>>(obs_slot, obs_kp, ids, n_kp, kp_point);
  P2P_LAUNCH_OK();
  return 0;
}

int launch_sfm_query_rows(Arena& ar, const double* m4, long long M, const long long* offsets, int P,
                          const int* pair_img, int n_queries, double px, const int* qkp_of_ep,
                          const unsigned long long* qkp_key, const double* qkp_n, const double* q_intr,
                          const unsigned long long* kp_key, const double* kp_xy, const int* kp_point, long long n_kp,
                          const double* pts, double* rows, long long* q_offsets, cudaStream_t st) {
  const long long n = std::max(M, (long long)n_queries + 1);
  const size_t tmp = std::max(sort_bytes(n, false), scan_bytes(n));
  int rc = ar.reserve(2 * align_up(n * 8 + 16, 256) + 2 * align_up(n * 4 + 16, 256) + align_up(tmp + 16, 256) + 4096);
  if (rc) return rc;
  Carve c{(char*)ar.take(ar.cap - 1024)};
  auto* k0 = c.take<unsigned long long>(n);
  auto* k1 = c.take<unsigned long long>(n);
  int* ids = c.take<int>(n);
  int* qc = c.take<int>(n_queries + 1);
  void* t = c.take<char>(tmp);
  P2P_CUDA_OK(cudaMemsetAsync(qc, 0, (n_queries + 1) * sizeof(int), st));
  size_t tb;
  if (M > 0) {
    query_key_kernel<<<grid_of(M), kSfmThreads, 0, st>>>(m4, M, offsets, P, pair_img, px, qkp_of_ep, kp_key, kp_xy,
                                                         kp_point, n_kp, k0);
    P2P_LAUNCH_OK();
    tb = tmp;
    P2P_CUDA_OK(cub::DeviceRadixSort::SortKeys(t, tb, k0, k1, (int)M, 0, 64, st));
    head_flag_kernel<<<grid_of(M), kSfmThreads, 0, st>>>(k1, M, ids);
    P2P_LAUNCH_OK();
    tb = tmp;
    P2P_CUDA_OK(cub::DeviceScan::InclusiveSum(t, tb, ids, ids, (int)M, st));
    query_row_kernel<<<grid_of(M), kSfmThreads, 0, st>>>(k1, ids, M, qkp_key, qkp_n, q_intr, pts, rows, qc);
    P2P_LAUNCH_OK();
  }
  tb = tmp;
  P2P_CUDA_OK(cub::DeviceScan::InclusiveSum(t, tb, qc, qc, n_queries + 1, st));
  offsets_kernel<<<grid_of(n_queries + 1), kSfmThreads, 0, st>>>(qc, n_queries, q_offsets);
  P2P_LAUNCH_OK();
  return 0;
}

}  // namespace p2p
