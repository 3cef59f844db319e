// The per-pair statistics of the relative-pose evaluation (relpose.py) for a batch of pairs in one launch: the cosines
// of the rotation and translation-direction errors of an estimated pose against the ground truth, and the number of
// rows whose symmetric epipolar error under the ground-truth E lies below each threshold.  Integer counts, so the
// result does not depend on the order of the atomics or on the device.
#include "kernels.h"
#include "ransac_common.cuh"

namespace p2p {
namespace {

constexpr int kRelposeThreads = 256;

// Every fp64 product, sum and quotient below is rounded on its own (no fused multiply-add), in the order written, so
// that oracle/relpose_oracle.py restates it bit for bit.
__device__ __forceinline__ double clip1(double c) { return c > 1.0 ? 1.0 : (c < -1.0 ? -1.0 : c); }   // keeps NaN

// E = [t]x R (row-major): row 0 = -t2 R1 + t1 R2, row 1 = t2 R0 - t0 R2, row 2 = t0 R1 - t1 R0 (R_i: row i of R).
__device__ __forceinline__ void essential_from_pose(const double* Rt, double (&E)[9]) {
  const double* R = Rt;
  const double t0 = Rt[9], t1 = Rt[10], t2 = Rt[11];
#pragma unroll
  for (int j = 0; j < 3; ++j) {
    E[j] = __dsub_rn(__dmul_rn(t1, R[6 + j]), __dmul_rn(t2, R[3 + j]));
    E[3 + j] = __dsub_rn(__dmul_rn(t2, R[j]), __dmul_rn(t0, R[6 + j]));
    E[6 + j] = __dsub_rn(__dmul_rn(t0, R[3 + j]), __dmul_rn(t1, R[j]));
  }
}

// (a0 b0 + a1 b1) + a2 b2
__device__ __forceinline__ double dot3_rn(double a0, double a1, double a2, double b0, double b1, double b2) {
  return __dadd_rn(__dadd_rn(__dmul_rn(a0, b0), __dmul_rn(a1, b1)), __dmul_rn(a2, b2));
}

// One block per pair (blockIdx.x).  Each thread counts per threshold in registers, a warp sums its counts and lane 0
// adds them to shared memory; plain stores write the record, so it needs no zeroing.
__global__ void __launch_bounds__(kRelposeThreads) relpose_errors_kernel(PairBatch B, const double* __restrict__ intr,
                                                                         const double* __restrict__ Rt_gt,
                                                                         const double* __restrict__ Rt_est,
                                                                         const int* __restrict__ n_inliers,
                                                                         RelposeErrArgs a, double* __restrict__ out,
                                                                         int out_stride) {
  __shared__ int cnt[kMaxRelposeThresholds];
  const int tid = threadIdx.x, p = blockIdx.x, nt = a.n_thr;
  if (tid < kMaxRelposeThresholds) cnt[tid] = 0;
  const PairRange pr = pair_range(B, p);
  const int m = effective_rows(B, p, pr.n);
  const double* k = intr + 8 * (size_t)p;
  const double fx1 = k[0], fy1 = k[1], cx1 = k[2], cy1 = k[3], fx2 = k[4], fy2 = k[5], cx2 = k[6], cy2 = k[7];
  const double* gt = Rt_gt + 12 * (size_t)p;
  double E[9];
  essential_from_pose(gt, E);
  __syncthreads();
  int c[kMaxRelposeThresholds];
#pragma unroll
  for (int j = 0; j < kMaxRelposeThresholds; ++j) c[j] = 0;
  const double* rows = B.rows + pr.row0 * B.stride;
  for (int r = tid; r < m; r += kRelposeThreads) {
    const double* q = rows + (size_t)r * B.stride;
    const double u0 = __ddiv_rn(__dsub_rn(q[0], cx1), fx1), v0 = __ddiv_rn(__dsub_rn(q[1], cy1), fy1);
    const double u1 = __ddiv_rn(__dsub_rn(q[2], cx2), fx2), v1 = __ddiv_rn(__dsub_rn(q[3], cy2), fy2);
    const double l0 = dot3_rn(E[0], E[1], E[2], u0, v0, 1.0);          // E x0
    const double l1 = dot3_rn(E[3], E[4], E[5], u0, v0, 1.0);
    const double l2 = dot3_rn(E[6], E[7], E[8], u0, v0, 1.0);
    const double m0 = dot3_rn(E[0], E[3], E[6], u1, v1, 1.0);          // E^T x1
    const double m1 = dot3_rn(E[1], E[4], E[7], u1, v1, 1.0);
    const double num = dot3_rn(u1, v1, 1.0, l0, l1, l2);                 // x1^T E x0
    const double d0 = __dadd_rn(__dmul_rn(l0, l0), __dmul_rn(l1, l1));
    const double d1 = __dadd_rn(__dmul_rn(m0, m0), __dmul_rn(m1, m1));
    const double err = __dmul_rn(__dmul_rn(num, num), __dadd_rn(__ddiv_rn(1.0, d0), __ddiv_rn(1.0, d1)));
#pragma unroll
    for (int j = 0; j < kMaxRelposeThresholds; ++j) c[j] += (err < a.thr[j]) ? 1 : 0;
  }
#pragma unroll
  for (int j = 0; j < kMaxRelposeThresholds; ++j) {
    if (j < nt) {
      const int s = __reduce_add_sync(0xffffffffu, c[j]);
      if ((tid & 31) == 0 && s) atomicAdd(&cnt[j], s);
    }
  }
  double* rec = out + (size_t)p * out_stride;
  if (tid == 0) {
    // cos of the rotation error (tr(R_gt^T R) - 1) / 2 and of the translation-direction error t_gt . t / (|t_gt| |t|),
    // clipped to [-1, 1]; NaN when the pair has no estimate (inlier count <= 0)
    double cr = __longlong_as_double(0x7ff8000000000000ll), ct = cr;
    if (n_inliers[p] > 0) {
      const double* R = Rt_est + 12 * (size_t)p;
      double tr = 0.0;
      for (int j = 0; j < 9; ++j) tr = __dadd_rn(tr, __dmul_rn(gt[j], R[j]));
      cr = clip1(__ddiv_rn(__dsub_rn(tr, 1.0), 2.0));
      const double dot = dot3_rn(gt[9], gt[10], gt[11], R[9], R[10], R[11]);
      const double ng = __dsqrt_rn(dot3_rn(gt[9], gt[10], gt[11], gt[9], gt[10], gt[11]));
      const double ne = __dsqrt_rn(dot3_rn(R[9], R[10], R[11], R[9], R[10], R[11]));
      ct = clip1(__ddiv_rn(dot, __dmul_rn(ng, ne)));
    }
    rec[0] = cr;
    rec[1] = ct;
  }
  __syncthreads();
  int* counts = reinterpret_cast<int*>(rec + 2);
  if (tid < nt) counts[tid] = cnt[tid];
  if (tid == 0) counts[nt] = m;
}

}  // namespace

int launch_relpose_errors(const PairBatch& B, const double* intr, const double* Rt_gt, const double* Rt_est,
                          const int* n_inliers, const RelposeErrArgs& a, double* out, int out_stride, cudaStream_t st) {
  relpose_errors_kernel<<<B.pairs, kRelposeThreads, 0, st>>>(B, intr, Rt_gt, Rt_est, n_inliers, a, out, out_stride);
  P2P_LAUNCH_OK();
  return 0;
}

}  // namespace p2p
