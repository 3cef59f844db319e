// The image-overlap matrix of the reference's validation-pair precompute (utils/colmap/data_loading.py:54-70,
// cal_overlap_scores): for images i < j, |A_i ∩ A_j| / max(|A_i|, |A_j|) with A_i the indices of image i's keypoints
// whose point3D_id is > 0.  Each A_i becomes a bitset over keypoint indices, so the intersections are an integer Gram
// matrix of popcounts: exact in int32, and the final division is one IEEE fp64 division per entry, as Python's.
#include "kernels.h"

namespace p2p {
namespace {

constexpr int kPackThreads = 256;
constexpr int kTile = 64;               // images per tile side
constexpr int kChunk = 32;              // bitset words staged per step
constexpr int kCountThreads = 256;      // 16 x 16 threads, a 4 x 4 micro-tile each
constexpr int kMicro = kTile / 16;

// One block per image: warp w builds words w, w + 8, ... with one ballot per 32 keypoints (coalesced id reads), and
// the block's popcount sum is the image's count.  Words past the image's keypoints are zero.
__global__ void __launch_bounds__(kPackThreads) overlap_pack_kernel(const long long* __restrict__ ids,
                                                                    const long long* __restrict__ offsets, int words,
                                                                    unsigned* __restrict__ bits,
                                                                    int* __restrict__ counts) {
  __shared__ int total;
  const int img = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) total = 0;
  __syncthreads();
  const long long base = offsets[img];
  const long long n = min(max(offsets[img + 1] - base, 0LL), 32LL * words);   // defensive: the host checked both
  int c = 0;
  for (int w = warp; w < words; w += kPackThreads / 32) {
    const long long k = 32LL * w + lane;
    const unsigned word = __ballot_sync(0xffffffffu, k < n && ids[base + k] > 0);
    if (lane == 0) {
      bits[(size_t)img * words + w] = word;
      c += __popc(word);
    }
  }
  if (lane == 0 && c) atomicAdd(&total, c);
  __syncthreads();
  if (threadIdx.x == 0) counts[img] = total;
}

// (tile_i, tile_j) of linear block b over the upper triangle tile_i <= tile_j, row tile_j holding tile_j + 1 blocks.
__device__ __forceinline__ void tri_tile(int b, int& ti, int& tj) {
  int j = (int)((sqrt(8.0 * (double)b + 1.0) - 1.0) * 0.5);
  while ((long long)j * (j + 1) / 2 > b) --j;
  while ((long long)(j + 1) * (j + 2) / 2 <= b) ++j;
  tj = j;
  ti = b - (int)((long long)j * (j + 1) / 2);
}

// One block per tile pair tile_i <= tile_j of the upper triangle.  Word chunks of both tiles are staged transposed in
// shared memory ([word][image], one pad column against bank conflicts); thread (ty, tx) owns rows ty + 16u and columns
// tx + 16v.  The epilogue writes every entry of the tile, and for tile_i < tile_j the zeros of the mirrored tile, so
// the whole [n, n] matrix is written and nothing depends on what the buffer held.
__global__ void __launch_bounds__(kCountThreads) overlap_count_kernel(const unsigned* __restrict__ bits, int n,
                                                                      int words, const int* __restrict__ counts,
                                                                      double* __restrict__ scores) {
  __shared__ unsigned sa[kChunk][kTile + 1];
  __shared__ unsigned sb[kChunk][kTile + 1];
  int ti, tj;
  tri_tile(blockIdx.x, ti, tj);
  const int i0 = ti * kTile, j0 = tj * kTile;
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  int acc[kMicro][kMicro] = {};
  for (int w0 = 0; w0 < words; w0 += kChunk) {
    // each warp loads 32 consecutive words of one image: a 128-byte row segment
    for (int e = threadIdx.x; e < kTile * kChunk; e += kCountThreads) {
      const int r = e / kChunk, k = e % kChunk, w = w0 + k;
      const bool wk = w < words;
      sa[k][r] = (wk && i0 + r < n) ? bits[(size_t)(i0 + r) * words + w] : 0u;
      sb[k][r] = (wk && j0 + r < n) ? bits[(size_t)(j0 + r) * words + w] : 0u;
    }
    __syncthreads();
#pragma unroll 4
    for (int k = 0; k < kChunk; ++k) {
      unsigned a[kMicro], b[kMicro];
#pragma unroll
      for (int u = 0; u < kMicro; ++u) {
        a[u] = sa[k][ty + 16 * u];
        b[u] = sb[k][tx + 16 * u];
      }
#pragma unroll
      for (int u = 0; u < kMicro; ++u)
#pragma unroll
        for (int v = 0; v < kMicro; ++v) acc[u][v] += __popc(a[u] & b[v]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int u = 0; u < kMicro; ++u) {
    const int i = i0 + ty + 16 * u;
    if (i >= n) continue;
    const int ni = counts[i];
#pragma unroll
    for (int v = 0; v < kMicro; ++v) {
      const int j = j0 + tx + 16 * v;
      if (j >= n) continue;
      double s;
      if (i < j) s = (double)acc[u][v] / (double)max(ni, counts[j]);
      else s = i == j ? 1.0 : 0.0;
      scores[(size_t)i * n + j] = s;
    }
  }
  if (ti != tj) {                       // the mirrored tile (tile_j, tile_i) lies below the diagonal
#pragma unroll
    for (int u = 0; u < kMicro; ++u) {
      const int i = j0 + ty + 16 * u;
      if (i >= n) continue;
#pragma unroll
      for (int v = 0; v < kMicro; ++v) scores[(size_t)i * n + i0 + tx + 16 * v] = 0.0;
    }
  }
}

}  // namespace

int launch_overlap_scores(const long long* ids, const long long* offsets, int n, int words, unsigned* bits,
                          int* counts, double* scores, cudaStream_t st) {
  if (n == 0) return 0;
  overlap_pack_kernel<<<n, kPackThreads, 0, st>>>(ids, offsets, words, bits, counts);
  P2P_LAUNCH_OK();
  const long long tiles = (n + kTile - 1) / kTile;
  overlap_count_kernel<<<(unsigned)(tiles * (tiles + 1) / 2), kCountThreads, 0, st>>>(bits, n, words, counts, scores);
  P2P_LAUNCH_OK();
  return 0;
}

}  // namespace p2p
