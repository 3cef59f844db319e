// SuperPoint's post-network steps and exact nearest-neighbour matching of descriptor sets (semantics in
// include/p2p_b200.h, p2p_sp_* and p2p_match_descriptors_batch; the restatement in oracle/superpoint_oracle.py).
//
//   keypoints    score kernel: softmax over 65 logits per cell, dustbin dropped, depth-to-space into [B][8Hc][8Wc];
//                NMS: five tiled (2r+1)^2 max-pool passes (init, then twice dilate + update) over that map;
//                candidates ((M ? s : 0) > threshold, inside the border) compacted in flat-index order by CUB's select,
//                so each image's run is row-major; top-k: per-image segmented radix sort of unique 64-bit keys
//                score_bits << 32 | ~index (descending), so exact score ties keep the lowest flat index
//   descriptors  cells L2-normalised into a [B][Hc*Wc][D] map, then one warp per keypoint: bilinear weights and sums
//                in fp64, renormalisation
//   matching     the defined similarity is the float64 fma chain over k = 0..D-1 of the (exact) fp32 x fp32 products.
//                Default: 3-pass fp16 hi/lo similarities on the tensor cores (wgmma) with each row's top 2 kept in
//                registers, then every row / column whose decision lies within 2 eps (DESIGN.md) redone in float64 on
//                the CUDA cores, so the result equals the float64 definition exactly.  match_impl 0: 64 x 64 float64
//                tiles for every similarity.  Mutual matching runs the row kernel with the sides swapped for the
//                column argmax.  No float atomics: results are identical across runs, and per pair across batches.
#include <cub/cub.cuh>
#include <thrust/iterator/counting_iterator.h>

#include "common.cuh"
#include "kernels.h"
#include "umma_ptx.cuh"

namespace p2p {
namespace {

constexpr int kPoolTile = 32;                              // output tile of the max-pool passes
constexpr int kPoolIn = kPoolTile + 2 * kSpMaxNmsRadius;   // input tile with halo
constexpr int kMatchTile = 64;                             // rows x columns per block of the similarity kernel
constexpr int kMatchK = 16;                                // k chunk staged in shared memory

// ---- keypoints ------------------------------------------------------------------------------------------------------
__global__ void sp_score_kernel(const float* __restrict__ logits, int B, int Hc, int Wc, float* __restrict__ smap) {
  const long long cell = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long HWc = (long long)Hc * Wc;
  if (cell >= B * HWc) return;
  const int b = (int)(cell / HWc);
  const int q = (int)(cell - b * HWc);
  const int cy = q / Wc, cx = q - cy * Wc;
  const float* x = logits + (long long)b * 65 * HWc + q;
  float m = -INFINITY;
  for (int c = 0; c < 65; ++c) m = fmaxf(m, x[c * HWc]);
  float sum = 0.f;
  for (int c = 0; c < 65; ++c) sum += expf(x[c * HWc] - m);
  const int W = Wc * 8;
  float* out = smap + (long long)b * HWc * 64 + (long long)(cy * 8) * W + cx * 8;
  for (int c = 0; c < 64; ++c) out[(c >> 3) * W + (c & 7)] = expf(x[c * HWc] - m) / sum;
}

// One (2r+1)^2 max-pool pass of the NMS, out-of-image taps never win.
//   MODE 0: m_out = (s == maxpool(s))
//   MODE 1: m_out = maxpool(m_in) > 0                                   (the suppression mask S)
//   MODE 2: v = m_in ? 0 : s;  m_out |= (v == maxpool(v)) & !m_in       (m_in = S, m_out = M, updated in place)
template <int MODE>
__global__ void __launch_bounds__(256) sp_pool_kernel(const float* __restrict__ smap, const uint8_t* __restrict__ m_in,
                                                      uint8_t* __restrict__ m_out, int H, int W, int r) {
  __shared__ float tile[kPoolIn][kPoolIn + 1];
  __shared__ float rowmax[kPoolIn][kPoolTile + 1];
  const int b = blockIdx.z;
  const long long base = (long long)b * H * W;
  const int x0 = blockIdx.x * kPoolTile - r, y0 = blockIdx.y * kPoolTile - r;
  const int n_in = kPoolTile + 2 * r;
  const int tid = threadIdx.y * blockDim.x + threadIdx.x;
  for (int i = tid; i < n_in * n_in; i += 256) {
    const int ty = i / n_in, tx = i - ty * n_in;
    const int y = y0 + ty, x = x0 + tx;
    float v = -INFINITY;
    if (y >= 0 && y < H && x >= 0 && x < W) {
      const long long p = base + (long long)y * W + x;
      if (MODE == 0) v = smap[p];
      else if (MODE == 1) v = m_in[p] ? 1.f : 0.f;
      else v = m_in[p] ? 0.f : smap[p];
    }
    tile[ty][tx] = v;
  }
  __syncthreads();
  for (int i = tid; i < n_in * kPoolTile; i += 256) {
    const int ty = i / kPoolTile, tx = i - ty * kPoolTile;
    float m = tile[ty][tx];
    for (int d = 1; d <= 2 * r; ++d) m = fmaxf(m, tile[ty][tx + d]);
    rowmax[ty][tx] = m;
  }
  __syncthreads();
  for (int i = tid; i < kPoolTile * kPoolTile; i += 256) {
    const int ty = i / kPoolTile, tx = i - ty * kPoolTile;
    const int y = blockIdx.y * kPoolTile + ty, x = blockIdx.x * kPoolTile + tx;
    if (y >= H || x >= W) continue;
    float m = rowmax[ty][tx];
    for (int d = 1; d <= 2 * r; ++d) m = fmaxf(m, rowmax[ty + d][tx]);
    const float c = tile[ty + r][tx + r];
    const long long p = base + (long long)y * W + x;
    if (MODE == 0) m_out[p] = c == m;
    else if (MODE == 1) m_out[p] = m > 0.f;
    else if (!m_in[p] && c == m) m_out[p] = 1;
  }
}

// the kept score (M ? s : 0), which is what a keypoint reports: non-maxima pass a negative threshold with score 0
__device__ __forceinline__ float kept_score(const float* smap, const uint8_t* M, int p) { return M[p] ? smap[p] : 0.f; }

struct KpCandidate {   // (M ? s : 0) > threshold, inside the border
  const float* smap;
  const uint8_t* M;
  int H, W, border;
  float thr;
  __device__ __forceinline__ bool operator()(int p) const {
    const int HW = H * W;
    const int q = p % HW;
    const int y = q / W, x = q - y * W;
    if (y < border || y >= H - border || x < border || x >= W - border) return false;
    return kept_score(smap, M, p) > thr;
  }
};

// seg[b] = first selected entry of image b (the selection is in flat-index order), seg[B] = n_sel
__global__ void sp_segments_kernel(const int* __restrict__ sel, const int* __restrict__ n_sel, int B, int HW,
                                   int* __restrict__ seg) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b > B) return;
  const int n = *n_sel;
  if (b == B) {
    seg[B] = n;
    return;
  }
  const int key = b * HW;
  int lo = 0, hi = n;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (sel[mid] < key) lo = mid + 1;
    else hi = mid;
  }
  seg[b] = lo;
}

__global__ void sp_sort_keys_kernel(const int* __restrict__ sel, const int* __restrict__ n_sel,
                                    const float* __restrict__ smap, const uint8_t* __restrict__ M, int HW,
                                    unsigned long long* __restrict__ keys) {
  const int n = *n_sel;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const int p = sel[i];
    keys[i] = (unsigned long long)__float_as_uint(kept_score(smap, M, p)) << 32 | (0xffffffffu - (unsigned)(p % HW));
  }
}

// counts[b] = first output row of image b, counts[B] = total (rows per image: all candidates, or the first k)
__global__ void sp_counts_kernel(const int* __restrict__ seg, int B, int k, long long* __restrict__ counts) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  long long o = 0;
  for (int b = 0; b < B; ++b) {
    counts[b] = o;
    const int n = seg[b + 1] - seg[b];
    o += k >= 0 ? min(n, k) : n;
  }
  counts[B] = o;
}

__global__ void sp_write_kernel(const int* __restrict__ idx, const int* __restrict__ seg, const long long* __restrict__ counts,
                                const int* __restrict__ n_sel, int B, int W, int HW, const float* __restrict__ smap,
                                const uint8_t* __restrict__ M, float* __restrict__ kp, float* __restrict__ kp_score) {
  const int n = *n_sel;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    int lo = 0, hi = B - 1;                       // image of entry i: the last b with seg[b] <= i
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (seg[mid] <= i) lo = mid;
      else hi = mid - 1;
    }
    const int b = lo;
    const long long rank = i - seg[b];
    const long long o = counts[b] + rank;
    if (o >= counts[b + 1]) continue;
    const int p = idx[i];
    const int q = p - b * HW;
    const int y = q / W;
    kp[2 * o] = (float)(q - y * W);
    kp[2 * o + 1] = (float)y;
    kp_score[o] = kept_score(smap, M, p);
  }
}

// ---- descriptors ----------------------------------------------------------------------------------------------------
// raw [B][D][Hc*Wc] -> out [B][Hc*Wc][D], each cell divided by max(|cell|, 1e-12) (F.normalize)
__global__ void sp_desc_normalize_kernel(const float* __restrict__ raw, int B, int D, int HWc, float* __restrict__ out) {
  const long long cell = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (cell >= (long long)B * HWc) return;
  const int b = (int)(cell / HWc);
  const int q = (int)(cell - (long long)b * HWc);
  const float* x = raw + (long long)b * D * HWc + q;
  double ss = 0.0;
  for (int c = 0; c < D; ++c) {
    const double v = x[(long long)c * HWc];
    ss += v * v;
  }
  const double inv = 1.0 / fmax(sqrt(ss), 1e-12);
  float* o = out + cell * D;
  for (int c = 0; c < D; ++c) o[c] = (float)(x[(long long)c * HWc] * inv);
}

// One warp per keypoint: grid_sample(align_corners=True, zero padding) at u = (x - 3.5) / (8 Wc - 4.5) * (Wc - 1)
// (and v likewise), then the result divided by max(|.|, 1e-12).
__global__ void sp_desc_sample_kernel(const float* __restrict__ nmap, const float* __restrict__ kp,
                                      const long long* __restrict__ kp_off, long long N, int B, int D, int Hc, int Wc,
                                      float* __restrict__ out) {
  const long long n = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (n >= N) return;
  int lo = 0, hi = B - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (kp_off[mid] <= n) lo = mid;
    else hi = mid - 1;
  }
  const int b = lo;
  const double gx = ((double)kp[2 * n] - 3.5) / (8.0 * Wc - 4.5) * 2.0 - 1.0;
  const double gy = ((double)kp[2 * n + 1] - 3.5) / (8.0 * Hc - 4.5) * 2.0 - 1.0;
  const double ix = (gx + 1.0) * 0.5 * (Wc - 1), iy = (gy + 1.0) * 0.5 * (Hc - 1);
  const double fx = floor(ix), fy = floor(iy);
  const int x0 = (int)fx, y0 = (int)fy;
  const double ax = ix - fx, ay = iy - fy;
  const double w[4] = {(1.0 - ax) * (1.0 - ay), ax * (1.0 - ay), (1.0 - ax) * ay, ax * ay};
  const int cx[4] = {x0, x0 + 1, x0, x0 + 1}, cy[4] = {y0, y0, y0 + 1, y0 + 1};
  const float* src[4];
  for (int t = 0; t < 4; ++t)
    src[t] = (cx[t] >= 0 && cx[t] < Wc && cy[t] >= 0 && cy[t] < Hc)
                 ? nmap + ((long long)b * Hc * Wc + (long long)cy[t] * Wc + cx[t]) * D
                 : nullptr;
  constexpr int kMaxPerLane = kSpMaxDescDim / 32;
  double acc[kMaxPerLane];
  double ss = 0.0;
#pragma unroll
  for (int j = 0; j < kMaxPerLane; ++j) {
    const int c = lane + 32 * j;
    double a = 0.0;
    if (c < D)
      for (int t = 0; t < 4; ++t)
        if (src[t]) a += w[t] * (double)src[t][c];
    acc[j] = a;
    ss += a * a;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
  const double inv = 1.0 / fmax(sqrt(ss), 1e-12);
#pragma unroll
  for (int j = 0; j < kMaxPerLane; ++j) {
    const int c = lane + 32 * j;
    if (c < D) out[n * D + c] = (float)(acc[j] * inv);
  }
}

// ---- matching -------------------------------------------------------------------------------------------------------
struct Top2 {
  double s1, s2;
  int j1;
};

// (s desc, index asc) total order: a merge that keeps the best two values and the best index is order-independent
__device__ __forceinline__ void top2_merge(Top2& a, double bs1, double bs2, int bj1) {
  if (bs1 > a.s1 || (bs1 == a.s1 && bj1 >= 0 && (a.j1 < 0 || bj1 < a.j1))) {
    a.s2 = fmax(bs2, a.s1);
    a.s1 = bs1;
    a.j1 = bj1;
  } else {
    a.s2 = fmax(a.s2, bs1);
  }
}

// Block (tile, pair): rows tile*64 .. +63 of side A of the pair against every column of side B.  Writes each row's
// best similarity, second-best similarity (-inf when the pair has one column) and best column (-1 with none).
__global__ void __launch_bounds__(256) sp_match_rows_kernel(const float* __restrict__ A, const float* __restrict__ Bm,
                                                            const long long* __restrict__ offA,
                                                            const long long* __restrict__ offB, int D,
                                                            double* __restrict__ s1_out, double* __restrict__ s2_out,
                                                            int* __restrict__ j1_out) {
  __shared__ double As[kMatchK][kMatchTile];
  __shared__ double Bs[kMatchK][kMatchTile];
  const int pair = blockIdx.y;
  const long long a0 = offA[pair], b0 = offB[pair];
  const int nA = (int)(offA[pair + 1] - a0), nB = (int)(offB[pair + 1] - b0);
  const int r0 = blockIdx.x * kMatchTile;
  if (r0 >= nA) return;
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  Top2 best[4];
#pragma unroll
  for (int r = 0; r < 4; ++r) best[r] = Top2{-INFINITY, -INFINITY, -1};
  for (int c0 = 0; c0 < nB; c0 += kMatchTile) {
    double acc[4][4];
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
      for (int c = 0; c < 4; ++c) acc[r][c] = 0.0;
    for (int k0 = 0; k0 < D; k0 += kMatchK) {
      __syncthreads();
      for (int i = tid; i < kMatchTile * kMatchK; i += 256) {
        const int row = i / kMatchK, k = i - row * kMatchK;
        As[k][row] = r0 + row < nA ? (double)A[(a0 + r0 + row) * D + k0 + k] : 0.0;
        Bs[k][row] = c0 + row < nB ? (double)Bm[(b0 + c0 + row) * D + k0 + k] : 0.0;
      }
      __syncthreads();
#pragma unroll
      for (int k = 0; k < kMatchK; ++k) {
        double a[4], b[4];
#pragma unroll
        for (int r = 0; r < 4; ++r) a[r] = As[k][ty + 16 * r];
#pragma unroll
        for (int c = 0; c < 4; ++c) b[c] = Bs[k][tx + 16 * c];
#pragma unroll
        for (int r = 0; r < 4; ++r)
#pragma unroll
          for (int c = 0; c < 4; ++c) acc[r][c] = fma(a[r], b[c], acc[r][c]);   // the product is exact in fp64
      }
    }
    // columns in ascending order per thread: a strict > keeps the lowest index of a tie as the best
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const int j = c0 + tx + 16 * c;
      if (j >= nB) continue;
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        const double v = acc[r][c];
        if (v > best[r].s1) {
          best[r].s2 = best[r].s1;
          best[r].s1 = v;
          best[r].j1 = j;
        } else if (v > best[r].s2) {
          best[r].s2 = v;
        }
      }
    }
  }
#pragma unroll
  for (int r = 0; r < 4; ++r) {
#pragma unroll
    for (int o = 8; o > 0; o >>= 1) {
      const double s1 = __shfl_xor_sync(0xffffffffu, best[r].s1, o);
      const double s2 = __shfl_xor_sync(0xffffffffu, best[r].s2, o);
      const int j1 = __shfl_xor_sync(0xffffffffu, best[r].j1, o);
      top2_merge(best[r], s1, s2, j1);
    }
    const int row = r0 + ty + 16 * r;
    if (tx == 0 && row < nA) {
      s1_out[a0 + row] = best[r].s1;
      if (s2_out) s2_out[a0 + row] = best[r].s2;
      j1_out[a0 + row] = best[r].j1;
    }
  }
}

struct MatchRule {
  int mutual, has_min, has_ratio;
  double min_sim, ratio2;
};

__global__ void sp_match_finalize_kernel(const long long* __restrict__ off0, const long long* __restrict__ off1,
                                         const double* __restrict__ s1, const double* __restrict__ s2,
                                         const int* __restrict__ j1, const int* __restrict__ col_best, MatchRule rule,
                                         int* __restrict__ match, double* __restrict__ sim) {
  const int pair = blockIdx.y;
  const long long a0 = off0[pair], b0 = off1[pair];
  const int n = (int)(off0[pair + 1] - a0), m = (int)(off1[pair + 1] - b0);
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int j = j1[a0 + i];
  const double v = s1[a0 + i];
  bool ok = j >= 0;
  if (ok && rule.mutual) ok = col_best[b0 + j] == i;
  if (ok && rule.has_min) ok = v > rule.min_sim;
  if (ok && rule.has_ratio && m >= 2) ok = 1.0 - v < rule.ratio2 * (1.0 - s2[a0 + i]);
  match[a0 + i] = ok ? j : -1;
  sim[a0 + i] = ok ? v : 0.0;
}

// ---- matching on the tensor cores: 3-pass fp16 hi/lo similarities, float64 fix-up of undecided rows / columns ------
constexpr int kTcTile = 128;      // rows x columns per block
constexpr int kTcTileBytes = kTcTile * 128;                // one 128-row x 64-half swizzled operand tile
constexpr int kTcSmem = 4 * kTcTileBytes + 1024;           // A hi, A lo, B hi, B lo, plus alignment slack

// One warp per row: power-of-two scale 2^-e with max |x| 2^-e in [0.5, 1) (e >= -126), hi = fp16(x'), lo =
// fp16(x' - hi), and |x'| (fp32 sum of squares, rounded up by 2^-20 relative).
__global__ void sp_split_kernel(const float* __restrict__ x, long long n, int D, __half* __restrict__ hi,
                                __half* __restrict__ lo, int* __restrict__ expo, float* __restrict__ nrm) {
  const long long r = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (r >= n) return;
  const float* row = x + r * D;
  float m = 0.f;
  for (int c = lane; c < D; c += 32) m = fmaxf(m, fabsf(row[c]));
  m = warp_max(m);
  int e = 0;
  if (m > 0.f) frexpf(m, &e);
  e = max(e, -126);
  const float sc = ldexpf(1.f, -e);
  float ss = 0.f;
  for (int c = lane; c < D; c += 32) {
    const float v = row[c] * sc;
    const __half h = __float2half_rn(v);
    hi[r * D + c] = h;
    lo[r * D + c] = __float2half_rn(v - __half2float(h));
    ss += v * v;
  }
  ss = warp_sum(ss);
  if (lane == 0) {
    expo[r] = e;
    nrm[r] = sqrtf(ss) * (1.f + 0x1p-20f);
  }
}

// eps[pair] bounds |s_tc - s_fp64| of every (row, column) of the pair (DESIGN.md, "The tensor-core pass"):
//   eps = C1 U0 U1 + C2 sqrt(D) (U0 S1 + S0 U1) + C3 S0 S1,  U = max |x'| 2^e, S = max 2^e over each set
__global__ void sp_eps_kernel(const long long* __restrict__ off0, const long long* __restrict__ off1,
                              const int* __restrict__ e0, const float* __restrict__ n0, const int* __restrict__ e1,
                              const float* __restrict__ n1, int D, double* __restrict__ eps) {
  __shared__ double red[4][256];
  const int pair = blockIdx.x, tid = threadIdx.x;
  double u[2] = {0.0, 0.0}, sx[2] = {0.0, 0.0};
  for (int side = 0; side < 2; ++side) {
    const long long* off = side ? off1 : off0;
    const int* e = side ? e1 : e0;
    const float* nr = side ? n1 : n0;
    for (long long i = off[pair] + tid; i < off[pair + 1]; i += 256) {
      const double p = ldexp(1.0, e[i]);
      u[side] = fmax(u[side], (double)nr[i] * p);
      sx[side] = fmax(sx[side], p);
    }
  }
  red[0][tid] = u[0], red[1][tid] = u[1], red[2][tid] = sx[0], red[3][tid] = sx[1];
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (tid < o)
      for (int q = 0; q < 4; ++q) red[q][tid] = fmax(red[q][tid], red[q][tid + o]);
    __syncthreads();
  }
  if (tid == 0) {
    const double u22 = 0x1p-22, n_inst = 3.0 * D / 16.0;
    const double gamma = D * 0x1p-53 / (1.0 - D * 0x1p-53);
    const double C1 = (3.0 * u22 + n_inst * u22 * (1.0 + 0x1p-9) + gamma + 0x1p-23) * (1.0 + 0x1p-10);
    const double C2 = 0x1p-25 * (1.0 + 0x1p-8) * (1.0 + n_inst * u22);
    const double C3 = 2.0 * D * 0x1p-50;
    eps[pair] = C1 * red[0][0] * red[1][0] + C2 * sqrt((double)D) * (red[0][0] * red[3][0] + red[2][0] * red[1][0]) +
                C3 * red[2][0] * red[3][0];
  }
}

__device__ __forceinline__ void top2_push(Top2& t, double v, int j) {
  if (v > t.s1) {
    t.s2 = t.s1;
    t.s1 = v;
    t.j1 = j;
  } else if (v > t.s2) {
    t.s2 = v;
  }
}

// Block (tile, pair): rows tile*128 .. +127 of side A against every column of side B on the tensor cores: two
// warpgroups, each wgmma m64n128k16 (fp32 accumulate) over its 64 rows, passes hi*hi + hi*lo + lo*hi in one
// accumulator chain over k.  Operands are staged per 64-wide k chunk in 128-byte-swizzled K-major tiles (the layout
// make_sw128_desc describes).  Each row's approximate best, second best and best column.
__global__ void __launch_bounds__(256) sp_tc_top2_kernel(const __half* __restrict__ Ahi, const __half* __restrict__ Alo,
                                                         const int* __restrict__ Ae, const long long* __restrict__ offA,
                                                         const __half* __restrict__ Bhi,
                                                         const __half* __restrict__ Blo, const int* __restrict__ Be,
                                                         const long long* __restrict__ offB, int D,
                                                         double* __restrict__ s1_out, double* __restrict__ s2_out,
                                                         int* __restrict__ j1_out) {
  extern __shared__ __align__(1024) unsigned char tc_smem[];
  __shared__ int be_s[kTcTile];
  const int pair = blockIdx.y;
  const long long a0 = offA[pair], b0 = offB[pair];
  const int nA = (int)(offA[pair + 1] - a0), nB = (int)(offB[pair + 1] - b0);
  const int r0 = blockIdx.x * kTcTile;
  if (r0 >= nA) return;
  unsigned char* base = (unsigned char*)(((uintptr_t)tc_smem + 1023) & ~(uintptr_t)1023);
  const uint32_t sbase = smem_u32(base);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, wg = warpgroup_index();
  const int g = lane >> 2, t = lane & 3;
  const int rl[2] = {wg * 64 + (warp & 3) * 16 + g, wg * 64 + (warp & 3) * 16 + g + 8};
  int ea[2];
  Top2 best[2];
#pragma unroll
  for (int q = 0; q < 2; ++q) {
    ea[q] = r0 + rl[q] < nA ? Ae[a0 + r0 + rl[q]] : 0;
    best[q] = Top2{-INFINITY, -INFINITY, -1};
  }
  for (int c0 = 0; c0 < nB; c0 += kTcTile) {
    float acc[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = 0.f;
    for (int k0 = 0; k0 < D; k0 += 64) {
      __syncthreads();                                  // the previous chunk's wgmma has completed (waited below)
      for (int i = tid; i < 4 * kTcTile * 8; i += 256) {   // 4 tiles x 128 rows x 8 vectors of 8 halves
        const int arr = i >> 10, row = (i >> 3) & 127, v = i & 7;
        const bool isA = arr < 2;
        const int gr = (isA ? r0 : c0) + row;
        uint4 val = make_uint4(0, 0, 0, 0);
        if (gr < (isA ? nA : nB) && k0 + v * 8 < D) {
          const __half* src = arr == 0 ? Ahi : arr == 1 ? Alo : arr == 2 ? Bhi : Blo;
          val = *reinterpret_cast<const uint4*>(src + ((isA ? a0 : b0) + gr) * D + k0 + v * 8);
        }
        *reinterpret_cast<uint4*>(base + arr * kTcTileBytes + row * 128 + ((v ^ (row & 7)) << 4)) = val;
      }
      if (k0 == 0 && tid < kTcTile) be_s[tid] = c0 + tid < nB ? Be[b0 + c0 + tid] : 0;
      fence_proxy_async();                              // generic-proxy stores -> visible to wgmma
      __syncthreads();
      wgmma_fence();
      wgmma_fence_regs<64>(acc);
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {
        const uint32_t off = (uint32_t)kk * 32;
        const uint64_t ah = make_sw128_desc(sbase + 0 * kTcTileBytes + wg * 8192 + off);
        const uint64_t al = make_sw128_desc(sbase + 1 * kTcTileBytes + wg * 8192 + off);
        const uint64_t bh = make_sw128_desc(sbase + 2 * kTcTileBytes + off);
        const uint64_t bl = make_sw128_desc(sbase + 3 * kTcTileBytes + off);
        wgmma_f16<128>(acc, ah, bh, 1);
        wgmma_f16<128>(acc, ah, bl, 1);
        wgmma_f16<128>(acc, al, bh, 1);
      }
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_regs<64>(acc);
    }
    // accumulator layout of m64nNk16: acc[4j + 2h + c] is row g + 8h, column 8j + 2t + c of the warp's 16 rows
#pragma unroll
    for (int jb = 0; jb < 16; ++jb)
#pragma unroll
      for (int c = 0; c < 2; ++c) {
        const int jl = jb * 8 + 2 * t + c, j = c0 + jl;
        if (j >= nB) continue;
#pragma unroll
        for (int h = 0; h < 2; ++h) top2_push(best[h], ldexp((double)acc[4 * jb + 2 * h + c], ea[h] + be_s[jl]), j);
      }
  }
#pragma unroll
  for (int q = 0; q < 2; ++q) {
#pragma unroll
    for (int o = 1; o <= 2; o <<= 1) {
      const double s1 = __shfl_xor_sync(0xffffffffu, best[q].s1, o);
      const double s2 = __shfl_xor_sync(0xffffffffu, best[q].s2, o);
      const int j1 = __shfl_xor_sync(0xffffffffu, best[q].j1, o);
      top2_merge(best[q], s1, s2, j1);
    }
    if (t == 0 && r0 + rl[q] < nA) {
      s1_out[a0 + r0 + rl[q]] = best[q].s1;
      s2_out[a0 + r0 + rl[q]] = best[q].s2;
      j1_out[a0 + r0 + rl[q]] = best[q].j1;
    }
  }
}

// The defined similarity: float64 fma chain over k = 0 .. D-1 of the exact fp32 products.
__device__ __forceinline__ double dot64(const float* __restrict__ a, const float* __restrict__ b, int D) {
  double s = 0.0;
  for (int k = 0; k < D; ++k) s = fma((double)a[k], (double)b[k], s);
  return s;
}

// Rows (side 0): the best column is decided when the tensor-core margin s1 - s2 exceeds 2 eps (or there are fewer
// than 2 columns); then s1 is recomputed exactly, and the ratio test is decided when it gives the same answer at
// s2 - eps and s2 + eps (the float64 test is monotone in s2).  Anything else is flagged for the fix-up.  Columns
// (mutual, side 1 against side 0): decided when their margin exceeds 2 eps.
__global__ void sp_classify_kernel(const float* __restrict__ A, const float* __restrict__ Bm,
                                   const long long* __restrict__ offA, const long long* __restrict__ offB,
                                   const double* __restrict__ eps, int D, int is_row, int has_ratio, double ratio2,
                                   const double* __restrict__ s1t, const double* __restrict__ s2t,
                                   const int* __restrict__ j1, double* __restrict__ s1x, uint8_t* __restrict__ flag,
                                   double* __restrict__ tc_sim, int* __restrict__ tc_idx) {
  const int pair = blockIdx.y;
  const long long a0 = offA[pair], b0 = offB[pair];
  const int n = (int)(offA[pair + 1] - a0), m = (int)(offB[pair + 1] - b0);
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const long long gi = a0 + i;
  if (m == 0) {
    flag[gi] = 0;
    if (is_row) s1x[gi] = 0.0;
    return;
  }
  const double e = eps[pair];
  bool sure = m == 1 || s1t[gi] - s2t[gi] > 2.0 * e;
  if (is_row) {
    const int j = j1[gi];
    const double v = dot64(A + gi * D, Bm + (b0 + j) * D, D);
    s1x[gi] = v;
    if (tc_sim) tc_sim[gi] = s1t[gi], tc_idx[gi] = j;
    if (sure && has_ratio && m >= 2) {
      const bool lo = 1.0 - v < ratio2 * (1.0 - (s2t[gi] - e));
      const bool hi = 1.0 - v < ratio2 * (1.0 - (s2t[gi] + e));
      sure = lo == hi;
    }
  }
  flag[gi] = !sure;
}

// Exact float64 decision for one flagged row of side A: every column's defined similarity, best / second best / best
// column with ties to the lowest index.  One block per flagged row (grid-stride over the device count).
__global__ void __launch_bounds__(256, 1) sp_fixup_kernel(const float* __restrict__ A, const float* __restrict__ Bm,
                                                       const long long* __restrict__ offA,
                                                       const long long* __restrict__ offB, int K, int D,
                                                       const int* __restrict__ list, const int* __restrict__ count,
                                                       double* __restrict__ s1x, double* __restrict__ s2,
                                                       int* __restrict__ j1) {
  __shared__ float a_s[kMatchMaxDim];
  __shared__ double r1[8], r2[8];
  __shared__ int rj[8];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int cnt = *count;
  for (int f = blockIdx.x; f < cnt; f += gridDim.x) {
    const long long gi = list[f];
    int lo = 0, hi = K - 1;                // pair of row gi: the last p with offA[p] <= gi
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (offA[mid] <= gi) lo = mid;
      else hi = mid - 1;
    }
    const long long b0 = offB[lo];
    const int m = (int)(offB[lo + 1] - b0);
    __syncthreads();
    for (int k = tid; k < D; k += 256) a_s[k] = A[gi * D + k];
    __syncthreads();
    Top2 b{-INFINITY, -INFINITY, -1};
    for (int j = tid; j < m; j += 256) {
      const float* bj = Bm + (b0 + j) * D;
      double v = 0.0;
      for (int k = 0; k < D; ++k) v = fma((double)a_s[k], (double)bj[k], v);
      top2_push(b, v, j);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const double s1 = __shfl_xor_sync(0xffffffffu, b.s1, o);
      const double ss = __shfl_xor_sync(0xffffffffu, b.s2, o);
      const int jj = __shfl_xor_sync(0xffffffffu, b.j1, o);
      top2_merge(b, s1, ss, jj);
    }
    if (lane == 0) r1[warp] = b.s1, r2[warp] = b.s2, rj[warp] = b.j1;
    __syncthreads();
    if (tid == 0) {
      for (int w = 1; w < 8; ++w) top2_merge(b, r1[w], r2[w], rj[w]);
      s1x[gi] = b.s1;
      if (s2) s2[gi] = b.s2;
      j1[gi] = b.j1;
    }
  }
}

__global__ void sp_tc_finalize_kernel(const long long* __restrict__ off0, const long long* __restrict__ off1,
                                      const double* __restrict__ s1x, const double* __restrict__ s2,
                                      const int* __restrict__ j1, const int* __restrict__ col_best, MatchRule rule,
                                      int* __restrict__ match, double* __restrict__ sim) {
  const int pair = blockIdx.y;
  const long long a0 = off0[pair], b0 = off1[pair];
  const int n = (int)(off0[pair + 1] - a0), m = (int)(off1[pair + 1] - b0);
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int j = m > 0 ? j1[a0 + i] : -1;
  const double v = s1x[a0 + i];
  bool ok = j >= 0;
  if (ok && rule.mutual) ok = col_best[b0 + j] == i;
  if (ok && rule.has_min) ok = v > rule.min_sim;
  if (ok && rule.has_ratio && m >= 2) ok = 1.0 - v < rule.ratio2 * (1.0 - s2[a0 + i]);
  match[a0 + i] = ok ? j : -1;
  sim[a0 + i] = ok ? v : 0.0;
}

}  // namespace

// ---- host -----------------------------------------------------------------------------------------------------------
int launch_sp_keypoints(Arena& ar, const float* logits, int B, int Hc, int Wc, int r, float thr, int border, int k,
                        float* smap_out, float* kp, float* kp_score, long long* counts, cudaStream_t st) {
  const int H = Hc * 8, W = Wc * 8, HW = H * W;
  const int total = B * HW;
  size_t sel_b = 0, sort_b = 0;
  cub::DeviceSelect::If(nullptr, sel_b, thrust::counting_iterator<int>(0), (int*)nullptr, (int*)nullptr, total,
                        KpCandidate{});
  if (k >= 0)
    cub::DeviceSegmentedRadixSort::SortPairsDescending(nullptr, sort_b, (unsigned long long*)nullptr,
                                                       (unsigned long long*)nullptr, (int*)nullptr, (int*)nullptr,
                                                       total, B, (int*)nullptr, (int*)nullptr);
  const size_t n = (size_t)total;
  const size_t bytes = (smap_out ? 0 : n * 4) + 2 * n + n * 4 * (k >= 0 ? 2 : 1) + (k >= 0 ? n * 16 : 0) +
                       std::max(sel_b, sort_b) + (size_t)(B + 2) * 8 + 16 * 256;
  int rc = ar.reserve(bytes);
  if (rc) return rc;
  Carve cv{(char*)ar.take(bytes - 1024)};
  float* smap = smap_out ? smap_out : cv.take<float>(n);
  uint8_t* M = cv.take<uint8_t>(n);
  uint8_t* S = cv.take<uint8_t>(n);
  int* sel = cv.take<int>(n);
  int* n_sel = cv.take<int>(1);
  int* seg = cv.take<int>(B + 1);
  void* tmp = cv.take<char>(std::max(sel_b, sort_b));

  const long long cells = (long long)B * Hc * Wc;
  sp_score_kernel<<<(unsigned)cdiv(cells, 128), 128, 0, st>>>(logits, B, Hc, Wc, smap);
  P2P_LAUNCH_OK();
  const dim3 pg(cdiv(W, kPoolTile), cdiv(H, kPoolTile), B), pb(32, 8);
  sp_pool_kernel<0><<<pg, pb, 0, st>>>(smap, nullptr, M, H, W, r);
  P2P_LAUNCH_OK();
  for (int it = 0; it < 2; ++it) {
    sp_pool_kernel<1><<<pg, pb, 0, st>>>(smap, M, S, H, W, r);
    P2P_LAUNCH_OK();
    sp_pool_kernel<2><<<pg, pb, 0, st>>>(smap, S, M, H, W, r);
    P2P_LAUNCH_OK();
  }
  P2P_CUDA_OK(cub::DeviceSelect::If(tmp, sel_b, thrust::counting_iterator<int>(0), sel, n_sel, total,
                                    KpCandidate{smap, M, H, W, border, thr}, st));
  ++g_launch_count;
  sp_segments_kernel<<<cdiv(B + 1, 128), 128, 0, st>>>(sel, n_sel, B, HW, seg);
  P2P_LAUNCH_OK();
  const int* idx = sel;
  if (k >= 0) {
    unsigned long long* k0 = cv.take<unsigned long long>(n);
    unsigned long long* k1 = cv.take<unsigned long long>(n);
    int* v1 = cv.take<int>(n);
    const int wg = (int)std::min<long long>(cdiv(total, 256), 132 * 8);
    sp_sort_keys_kernel<<<wg, 256, 0, st>>>(sel, n_sel, smap, M, HW, k0);
    P2P_LAUNCH_OK();
    // segments are the images' runs of the selection; entries past seg[B] belong to no segment and are not read
    P2P_CUDA_OK(cub::DeviceSegmentedRadixSort::SortPairsDescending(tmp, sort_b, k0, k1, sel, v1, total, B, seg,
                                                                   seg + 1, 0, 64, st));
    ++g_launch_count;
    idx = v1;
  }
  sp_counts_kernel<<<1, 32, 0, st>>>(seg, B, k, counts);
  P2P_LAUNCH_OK();
  const int wg = (int)std::min<long long>(cdiv(total, 256), 132 * 8);
  sp_write_kernel<<<wg, 256, 0, st>>>(idx, seg, counts, n_sel, B, W, HW, smap, M, kp, kp_score);
  P2P_LAUNCH_OK();
  return 0;
}

int launch_sp_descriptors(Arena& ar, const float* raw, int B, int D, int Hc, int Wc, const float* kp,
                          const long long* kp_off, long long N, float* out, cudaStream_t st) {
  const size_t cells = (size_t)B * Hc * Wc;
  int rc = ar.reserve(cells * D * 4 + 1024);
  if (rc) return rc;
  float* nmap = (float*)ar.take(cells * D * 4);
  sp_desc_normalize_kernel<<<(unsigned)cdiv((long long)cells, 128), 128, 0, st>>>(raw, B, D, Hc * Wc, nmap);
  P2P_LAUNCH_OK();
  if (N == 0) return 0;
  sp_desc_sample_kernel<<<(unsigned)cdiv(N * 32, 256), 256, 0, st>>>(nmap, kp, kp_off, N, B, D, Hc, Wc, out);
  P2P_LAUNCH_OK();
  return 0;
}

static int match_fp64(Arena& ar, const float* d0, const float* d1, const long long* off0, const long long* off1,
                      int K, int D, int max_n0, int max_n1, long long n0, long long n1, const MatchRule& rule,
                      int* match, double* sim, cudaStream_t st) {
  const size_t bytes = (size_t)n0 * 20 + (size_t)n1 * 12 + 16 * 256;
  int rc = ar.reserve(bytes);
  if (rc) return rc;
  Carve cv{(char*)ar.take(bytes - 1024)};
  double* s1 = cv.take<double>(n0);
  double* s2 = cv.take<double>(n0);
  int* j1 = cv.take<int>(n0);
  double* cs1 = cv.take<double>(n1);
  int* col_best = cv.take<int>(n1);
  sp_match_rows_kernel<<<dim3(cdiv(max_n0, kMatchTile), K), 256, 0, st>>>(d0, d1, off0, off1, D, s1, s2, j1);
  P2P_LAUNCH_OK();
  if (rule.mutual && max_n1 > 0) {
    sp_match_rows_kernel<<<dim3(cdiv(max_n1, kMatchTile), K), 256, 0, st>>>(d1, d0, off1, off0, D, cs1, nullptr,
                                                                            col_best);
    P2P_LAUNCH_OK();
  }
  sp_match_finalize_kernel<<<dim3(cdiv(max_n0, 256), K), 256, 0, st>>>(off0, off1, s1, s2, j1, col_best, rule, match,
                                                                       sim);
  P2P_LAUNCH_OK();
  return 0;
}

int launch_match_descriptors(Arena& ar, const float* d0, const float* d1, const long long* off0,
                             const long long* off1, int K, int D, int max_n0, int max_n1, long long n0, long long n1,
                             int mutual, int has_min, double min_sim, int has_ratio, double ratio, int impl,
                             int* match, double* sim, double* tc_sim, int* tc_idx, double* eps_out,
                             int* n_fixed, cudaStream_t st) {
  const MatchRule rule{mutual, has_min, has_ratio, min_sim, ratio * ratio};
  if (max_n0 == 0) return 0;
  if (impl == 0) return match_fp64(ar, d0, d1, off0, off1, K, D, max_n0, max_n1, n0, n1, rule, match, sim, st);
  const long long nn = std::max(n0, n1);
  size_t sel_b = 0;
  cub::DeviceSelect::Flagged(nullptr, sel_b, thrust::counting_iterator<int>(0), (const uint8_t*)nullptr,
                             (int*)nullptr, (int*)nullptr, (int)nn);
  const size_t bytes = (size_t)(n0 + n1) * D * 4 + (size_t)(n0 + n1) * 8 + (size_t)n0 * 40 + (size_t)n1 * 25 +
                       (size_t)K * 8 + sel_b + 32 * 256;
  int rc = ar.reserve(bytes);
  if (rc) return rc;
  Carve cv{(char*)ar.take(bytes - 1024)};
  __half *h0 = cv.take<__half>(n0 * D), *l0 = cv.take<__half>(n0 * D);
  __half *h1 = cv.take<__half>(std::max(n1, 1ll) * D), *l1 = cv.take<__half>(std::max(n1, 1ll) * D);
  int *e0 = cv.take<int>(n0), *e1 = cv.take<int>(n1);
  float *nr0 = cv.take<float>(n0), *nr1 = cv.take<float>(n1);
  double* eps = eps_out ? eps_out : cv.take<double>(K);
  double *s1t = cv.take<double>(n0), *s2t = cv.take<double>(n0), *s1x = cv.take<double>(n0);
  int* j1 = cv.take<int>(n0);
  double *cs1 = cv.take<double>(n1), *cs2 = cv.take<double>(n1);
  int* cj1 = cv.take<int>(n1);
  uint8_t *f0 = cv.take<uint8_t>(n0), *f1 = cv.take<uint8_t>(n1);
  int *list = cv.take<int>(nn), *cnt = n_fixed ? n_fixed : cv.take<int>(2);
  void* tmp = cv.take<char>(sel_b);

  sp_split_kernel<<<(unsigned)cdiv(n0 * 32, 256), 256, 0, st>>>(d0, n0, D, h0, l0, e0, nr0);
  P2P_LAUNCH_OK();
  if (n1 > 0) {
    sp_split_kernel<<<(unsigned)cdiv(n1 * 32, 256), 256, 0, st>>>(d1, n1, D, h1, l1, e1, nr1);
    P2P_LAUNCH_OK();
  }
  sp_eps_kernel<<<K, 256, 0, st>>>(off0, off1, e0, nr0, e1, nr1, D, eps);
  P2P_LAUNCH_OK();
  P2P_ENSURE_SMEM(sp_tc_top2_kernel, kTcSmem);
  sp_tc_top2_kernel<<<dim3(cdiv(max_n0, kTcTile), K), 256, kTcSmem, st>>>(h0, l0, e0, off0, h1, l1, e1, off1, D, s1t, s2t,
                                                                    j1);
  P2P_LAUNCH_OK();
  sp_classify_kernel<<<dim3(cdiv(max_n0, 256), K), 256, 0, st>>>(d0, d1, off0, off1, eps, D, 1, has_ratio,
                                                                 rule.ratio2, s1t, s2t, j1, s1x, f0, tc_sim, tc_idx);
  P2P_LAUNCH_OK();
  P2P_CUDA_OK(cub::DeviceSelect::Flagged(tmp, sel_b, thrust::counting_iterator<int>(0), f0, list, cnt, (int)n0, st));
  ++g_launch_count;
  sp_fixup_kernel<<<132 * 4, 256, 0, st>>>(d0, d1, off0, off1, K, D, list, cnt, s1x, s2t, j1);
  P2P_LAUNCH_OK();
  if (mutual && max_n1 > 0) {
    sp_tc_top2_kernel<<<dim3(cdiv(max_n1, kTcTile), K), 256, kTcSmem, st>>>(h1, l1, e1, off1, h0, l0, e0, off0, D, cs1, cs2,
                                                                      cj1);
    P2P_LAUNCH_OK();
    sp_classify_kernel<<<dim3(cdiv(max_n1, 256), K), 256, 0, st>>>(d1, d0, off1, off0, eps, D, 0, 0, 0.0, cs1, cs2,
                                                                   cj1, nullptr, f1, nullptr, nullptr);
    P2P_LAUNCH_OK();
    P2P_CUDA_OK(cub::DeviceSelect::Flagged(tmp, sel_b, thrust::counting_iterator<int>(0), f1, list, cnt + 1, (int)n1,
                                           st));
    ++g_launch_count;
    sp_fixup_kernel<<<132 * 4, 256, 0, st>>>(d1, d0, off1, off0, K, D, list, cnt + 1, cs1, nullptr, cj1);
    P2P_LAUNCH_OK();
  } else {
    P2P_CUDA_OK(cudaMemsetAsync(cnt + 1, 0, sizeof(int), st));
  }
  sp_tc_finalize_kernel<<<dim3(cdiv(max_n0, 256), K), 256, 0, st>>>(off0, off1, s1x, s2t, j1, cj1, rule, match, sim);
  P2P_LAUNCH_OK();
  return 0;
}

}  // namespace p2p
