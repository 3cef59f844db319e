// Robust two-view model estimation on the device: RANSAC for a fundamental matrix (7-point minimal solver) or a homography
// (4-point DLT), with local optimisation; F with the DEGENSAC plane-degeneracy check (Chum, Werner & Matas, CVPR 2005);
// and the reference's Sampson distance (utils/eval/measure.py:18-40).
//
// One call enqueues, with no host sync:
//   verify_prep_kernel     (1 block)  effective row count, finiteness, Hartley normalisation, fp32 copy of the rows
//   verify_round_kernel<K> (x rounds) kRound hypotheses: minimal sample -> models (one thread each), then every
//                                     (model, row) pair scored in fp32 by warps over rows staged in shared memory
//   verify_select_kernel   (x rounds) best model so far (most inliers, ties to the lowest (hypothesis, root) index) and
//                                     the stopping bound log(1-conf) / log(1-w^s); later rounds return at once past it
//   verify_lo_kernel<K>    (1 block)  non-minimal refit on the winner's inliers while the count grows, final mask
// (verify_common.cuh, kind K = 0 for F and 1 for H, which share one prep and one select kernel; E runs the same
// kernels as kind 3 in pose.cu, and model 2, F with the DEGENSAC check, adds its launches to kind 0's in degensac.cu).
// A batch of pairs runs the same launches with the pair as grid dimension y: one block per pair for prep / select / LO,
// cdiv(count, 8) blocks per pair for a round; a pair past its stopping bound returns at once from later rounds.
// Every reduction runs in a fixed order and no grid size depends on the device, so results are bit-reproducible.
#include <math.h>

#include "kernels.h"
#include "verify_common.cuh"

namespace p2p {
namespace {

__global__ void sampson_kernel(const double* __restrict__ rows, int stride, int n, const double* __restrict__ F,
                               double* __restrict__ out) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n) return;
  double m[9];
#pragma unroll
  for (int j = 0; j < 9; ++j) m[j] = F[j];
  out[r] = sampson_distance(m, rows + (size_t)r * stride);
}

}  // namespace

size_t verify_scratch_bytes(int pairs, long long rows, bool rounds) { return scratch_bytes<0>(pairs, rows, rounds); }

int verify_chunk_pairs() { return chunk_pairs<0>(); }

int launch_find_model(int model, const PairBatch& B, double px_th, double conf, int max_iters, unsigned long long seed,
                      void* scratch, double* model_out, uint8_t* mask_out, int* count_out, cudaStream_t st) {
  if (model == 2)
    return launch_find_model_degensac(B, px_th, conf, max_iters, seed, scratch, model_out, mask_out, count_out, st);
  auto find = model == 0 ? find_model<0> : find_model<1>;
  return find(B, nullptr, {}, px_th, nullptr, conf, max_iters, seed, scratch, model_out, mask_out, count_out, st);
}

int launch_test_hypotheses(int model, const double* rows, int stride, int n, double px_th, unsigned long long seed,
                           int count, void* scratch, double* models_out, int* counts_out, cudaStream_t st) {
  auto test = model == 0 ? test_hypotheses<0> : test_hypotheses<1>;
  return test(rows, stride, n, {}, px_th, seed, count, scratch, models_out, counts_out, st);
}

int launch_sampson_distance(const double* rows, int stride, int n, const double* F, double* out, cudaStream_t st) {
  if (n == 0) return 0;
  sampson_kernel<<<cdiv(n, 256), 256, 0, st>>>(rows, stride, n, F, out);
  P2P_LAUNCH_OK();
  return 0;
}

}  // namespace p2p
