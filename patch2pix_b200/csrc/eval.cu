// The three Sampson-distance histograms of the reference's validation loop (utils/train/eval_epoch_immatch.py:62-91,
// binned as utils/eval/measure.py:115-141 does) in one launch: coarse and refined matches against the ground-truth F,
// and the refined ones under the E-RANSAC inlier mask.  Integer counts, so the result is bit-reproducible.
#include "kernels.h"
#include "ransac_common.cuh"

namespace p2p {
namespace {

// np.histogram(d, edges) bin of d, or -1: edges[i] <= d < edges[i+1], the last bin closed; NaN, inf and values outside
// the edges get -1.  With increasing edges, the number of edges[0 .. ne-2] at or below d is the bin + 1, and only the
// last bin needs the upper bound.
__device__ __forceinline__ int hist_bin(const EpiHistArgs& a, double d) {
  int b = -1;
#pragma unroll
  for (int i = 0; i < kMaxHistEdges - 1; ++i) b += (i < a.n_edges - 1 && d >= a.edges[i]) ? 1 : 0;
  return d <= a.edges[a.n_edges - 1] ? b : -1;
}

// One block: shared-memory integer counts over m = min(n, *n_dev) rows, then one plain store of all 3 x n_edges words,
// so counts_out needs no zeroing and the result does not depend on the launch order of the atomics.
__global__ void __launch_bounds__(kHistThreads) epipolar_hist_kernel(const double* __restrict__ rows, int stride, int n,
                                                                     const double* __restrict__ n_dev, int coarse_col,
                                                                     const uint8_t* __restrict__ mask, EpiHistArgs a,
                                                                     int* __restrict__ counts_out) {
  __shared__ int cnt[3][kMaxHistEdges];
  const int tid = threadIdx.x, ne = a.n_edges;
  if (tid < 3 * kMaxHistEdges) cnt[tid / kMaxHistEdges][tid % kMaxHistEdges] = 0;
  int m = n;
  if (n_dev != nullptr) {
    const double v = *n_dev;
    if (v >= 0.0 && v < (double)n) m = (int)v;
  }
  __syncthreads();
  int c_mask = 0;
  for (int r = tid; r < m; r += kHistThreads) {
    const double* p = rows + (size_t)r * stride;
    if (coarse_col >= 0) {
      const int b = hist_bin(a, sampson_distance(a.F, p + coarse_col));
      if (b >= 0) atomicAdd(&cnt[0][b], 1);
    }
    const int b = hist_bin(a, sampson_distance(a.F, p));
    if (b >= 0) atomicAdd(&cnt[1][b], 1);
    if (mask != nullptr && mask[r] != 0) {
      if (b >= 0) atomicAdd(&cnt[2][b], 1);
      ++c_mask;
    }
  }
  if (c_mask) atomicAdd(&cnt[2][ne - 1], c_mask);
  if (tid == 0) {                      // rows considered
    cnt[0][ne - 1] = coarse_col >= 0 ? m : 0;
    cnt[1][ne - 1] = m;
  }
  __syncthreads();
  if (tid < 3 * ne) counts_out[tid] = cnt[tid / ne][tid % ne];
}

}  // namespace

int launch_epipolar_histograms(const double* rows, int stride, int n, const double* n_dev, int coarse_col,
                               const uint8_t* mask, const EpiHistArgs& a, int* counts_out, cudaStream_t st) {
  epipolar_hist_kernel<<<1, kHistThreads, 0, st>>>(rows, stride, n, n_dev, coarse_col, mask, a, counts_out);
  P2P_LAUNCH_OK();
  return 0;
}

}  // namespace p2p
