// The per-pair statistics of the HPatches evaluation (hpatches.py) in one launch: reprojection-error counts against a
// ground-truth H at each threshold, and the corner error of an estimated H.  Integer counts, so the result is
// bit-reproducible.
#include "kernels.h"

namespace p2p {
namespace {

// pi(H [x, y, 1]^T) in fp64 with the products and sums rounded one at a time (no fused multiply-add), in the order
// (h0 x + h1 y) + h2, so that a numpy restatement of the same expression gives the same bits.  Returns w.
__device__ __forceinline__ double project_h(const double* H, double x, double y, double& px, double& py) {
  const double u = __dadd_rn(__dadd_rn(__dmul_rn(H[0], x), __dmul_rn(H[1], y)), H[2]);
  const double v = __dadd_rn(__dadd_rn(__dmul_rn(H[3], x), __dmul_rn(H[4], y)), H[5]);
  const double w = __dadd_rn(__dadd_rn(__dmul_rn(H[6], x), __dmul_rn(H[7], y)), H[8]);
  px = __ddiv_rn(u, w);
  py = __ddiv_rn(v, w);
  return w;
}

__device__ __forceinline__ double dist2d(double ax, double ay, double bx, double by) {
  const double dx = __dsub_rn(ax, bx), dy = __dsub_rn(ay, by);
  return __dsqrt_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)));
}

// One block.  Each thread keeps its own count per threshold in registers (d <= t_j; NaN and inf fail every test), a
// warp sums them and its lane 0 adds them to shared memory; one plain store writes counts_out, so it needs no zeroing
// and the result does not depend on the order of the atomics.  Thread 0 computes the corner error.
__global__ void __launch_bounds__(kHistThreads) homography_errors_kernel(const double* __restrict__ rows, int stride,
                                                                         int n, const double* __restrict__ n_dev,
                                                                         HomErrArgs a,
                                                                         const double* __restrict__ H_pred,
                                                                         int* __restrict__ counts_out,
                                                                         double* __restrict__ corner_err_out) {
  __shared__ int cnt[kMaxHomThresholds];
  const int tid = threadIdx.x, nt = a.n_thr;
  if (tid < kMaxHomThresholds) cnt[tid] = 0;
  int m = n;
  if (n_dev != nullptr) {
    const double v = *n_dev;
    if (v >= 0.0 && v < (double)n) m = (int)v;
  }
  __syncthreads();
  int c[kMaxHomThresholds];
#pragma unroll
  for (int j = 0; j < kMaxHomThresholds; ++j) c[j] = 0;
  for (int r = tid; r < m; r += kHistThreads) {
    const double* p = rows + (size_t)r * stride;
    double px, py;
    project_h(a.H, p[0], p[1], px, py);
    const double d = dist2d(px, py, p[2], p[3]);
#pragma unroll
    for (int j = 0; j < kMaxHomThresholds; ++j) c[j] += (d <= a.thr[j]) ? 1 : 0;
  }
#pragma unroll
  for (int j = 0; j < kMaxHomThresholds; ++j) {
    if (j < nt) {
      const int s = __reduce_add_sync(0xffffffffu, c[j]);
      if ((tid & 31) == 0 && s) atomicAdd(&cnt[j], s);
    }
  }
  if (tid == 0) {
    // corners of image 1 (its original size); +inf without a model, at a corner with w = 0, or when not finite
    const int count = reinterpret_cast<const int*>(H_pred + 9)[0];
    double err = HUGE_VAL;
    if (count > 0) {
      const double cx[4] = {0.0, (double)(a.width - 1), 0.0, (double)(a.width - 1)};
      const double cy[4] = {0.0, 0.0, (double)(a.height - 1), (double)(a.height - 1)};
      double sum = 0.0;
      bool ok = true;
      for (int k = 0; k < 4; ++k) {
        double gx, gy, ex, ey;
        const double wg = project_h(a.H, cx[k], cy[k], gx, gy);
        const double we = project_h(H_pred, cx[k], cy[k], ex, ey);
        ok = ok && wg != 0.0 && we != 0.0;
        sum = __dadd_rn(sum, dist2d(gx, gy, ex, ey));
      }
      const double e = __ddiv_rn(sum, 4.0);
      if (ok && isfinite(e)) err = e;
    }
    *corner_err_out = err;
  }
  __syncthreads();
  if (tid < nt) counts_out[tid] = cnt[tid];
  if (tid == 0) counts_out[nt] = m;
}

}  // namespace

int launch_homography_errors(const double* rows, int stride, int n, const double* n_dev, const HomErrArgs& a,
                             const double* H_pred, int* counts_out, double* corner_err_out, cudaStream_t st) {
  homography_errors_kernel<<<1, kHistThreads, 0, st>>>(rows, stride, n, n_dev, a, H_pred, counts_out, corner_err_out);
  P2P_LAUNCH_OK();
  return 0;
}

}  // namespace p2p
