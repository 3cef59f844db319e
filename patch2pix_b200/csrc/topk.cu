// Top-k matches of an NCNet correlation volume: the reference's corr_to_matches_topk
// (networks/ncn/extract_ncmatches.py:96-158) for a whole batch in one launch per direction.
//
// A slice is what one cell is matched against: forward (invert = 0) the column x[a * nB + s] of B cell s over all
// A cells a; inverted the row x[s * nB + b] of A cell s.  Each slice yields its k best cells, ranked by the raw fp32
// value, descending (softmax is monotone, so this is the order of the softmax scores too), exact ties broken by the
// lowest flat cell index -- the rule of proposals_dir*_kernel.  The order is therefore a total order on
// key = (f2ord(value) << 16) | (0xffff - index), a 48-bit integer that is unique within a slice; +0 and -0 are one
// value.
//
// One CTA takes G consecutive slices of one batch item (G = 8, 4, 2, 1 for slices of up to 4096, 8192, 16384,
// 32768 cells) and stages them in shared memory as 32-bit ordered values.  Forward, the G columns are read as rows of
// G adjacent floats; inverted, the G rows are one contiguous block.  A team of 512 / G threads then works on each
// slice, all teams in lockstep (every loop bound is the same for all of them, so block barriers serve as team
// barriers):
//   1. max and the fp32 softmax denominator sum exp(x - max), reduced in a fixed order;
//   2. ranks are produced in chunks of R (R = next power of two >= k, at most 8192 / G): a radix select over the
//      staged slice finds the key of the chunk's last rank, 8 bits per pass from the top (six passes, fewer when the
//      selected bin holds exactly the ranks still needed), with warp-aggregated shared-memory histograms (the ReLU at
//      the end of the NeighConsensus stack leaves many exact zeros, which would otherwise serialise on one bin);
//   3. the keys between the previous chunk's threshold and this one -- exactly the chunk's ranks -- are compacted and
//      bitonic-sorted in shared memory, then written out: rank-major forward (rank r of slice s at r * nSlices + s),
//      cell-major inverted (s * k + r), relocalised through the packed maxpool4d code as emit_match does, with score
//      exp(x - max) / sum, or x itself when do_softmax is 0.
// Nothing depends on the grid or on the batch size, so a batch gives bit for bit the results of single calls.
#include "kernels.h"

namespace p2p {
namespace {

constexpr int kTopkThreads = 512;
constexpr int kTopkMaxTeams = 8;

__device__ __forceinline__ unsigned long long topk_key(unsigned v, int i) {
  return ((unsigned long long)v << 16) | (unsigned)(0xffff - i);
}

// Max (unsigned) / sum (float) over a team of T threads; every thread of the block calls it, every thread gets its
// team's result.  Partials are combined in warp order, so the result is deterministic.
__device__ __forceinline__ unsigned team_max(unsigned v, unsigned* red, int g, int T) {
  v = __reduce_max_sync(0xffffffffu, v);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  const int W = T >> 5;
  unsigned r = 0;
  for (int w = 0; w < W; ++w) r = max(r, red[g * W + w]);
  __syncthreads();
  return r;
}

__device__ __forceinline__ float team_sum(float v, float* red, int g, int T) {
  v = warp_sum(v);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  const int W = T >> 5;
  float r = 0.f;
  for (int w = 0; w < W; ++w) r += red[g * W + w];
  __syncthreads();
  return r;
}

template <bool INVERT>
__global__ void __launch_bounds__(kTopkThreads, 2)
    corr_topk_kernel(const float* __restrict__ x, const uint8_t* __restrict__ code, int nA, int nB, int wA, int wB,
                     int G, int R, int k, int ks, int do_softmax, long long* __restrict__ jA_out,
                     long long* __restrict__ iA_out, long long* __restrict__ jB_out, long long* __restrict__ iB_out,
                     float* __restrict__ sc_out) {
  extern __shared__ __align__(16) unsigned char topk_smem[];
  __shared__ unsigned hist[kTopkMaxTeams][256];
  __shared__ unsigned long long s_prefix[kTopkMaxTeams];
  __shared__ unsigned s_rem[kTopkMaxTeams], s_ctr[kTopkMaxTeams], s_done[kTopkMaxTeams];
  __shared__ unsigned s_redu[kTopkThreads / 32];
  __shared__ float s_redf[kTopkThreads / 32];

  const int N = INVERT ? nB : nA;         // slice length
  const int ns = INVERT ? nA : nB;        // slices per batch item
  const int S = N + 1;                    // odd pitch: the column loads of G slices fall in G different banks
  const int T = kTopkThreads / G, g = threadIdx.x / T, lt = threadIdx.x - g * T;
  const int s0 = blockIdx.x * G;
  const size_t vol = (size_t)nA * nB;
  const float* xb = x + blockIdx.y * vol;
  unsigned long long* buf = reinterpret_cast<unsigned long long*>(topk_smem) + (size_t)g * R;
  unsigned* keys = reinterpret_cast<unsigned*>(reinterpret_cast<unsigned long long*>(topk_smem) + (size_t)G * R);

  // ---- stage the G slices (slices past the last one read as zeros and are never written) ----
  if (INVERT) {
    const size_t base = (size_t)s0 * nB, end = (size_t)ns * nB;
    for (int f = threadIdx.x; f < G * N; f += kTopkThreads) {
      const float v = base + f < end ? xb[base + f] : 0.f;
      keys[(f / N) * S + f % N] = f2ord(v == 0.f ? 0.f : v);
    }
  } else {
    const int lg = __ffs(G) - 1;
    for (int f = threadIdx.x; f < G * N; f += kTopkThreads) {
      const int gg = f & (G - 1), a = f >> lg;
      const float v = s0 + gg < ns ? xb[(size_t)a * nB + s0 + gg] : 0.f;
      keys[gg * S + a] = f2ord(v == 0.f ? 0.f : v);
    }
  }
  __syncthreads();
  const unsigned* kv = keys + g * S;

  // ---- 1. max and softmax denominator ----
  unsigned m = 0;
  for (int i = lt; i < N; i += T) m = max(m, kv[i]);
  const float mx = ord2f(team_max(m, s_redu, g, T));
  float sum = 1.f;
  if (do_softmax) {
    float s = 0.f;
    for (int i = lt; i < N; i += T) s += expf(ord2f(kv[i]) - mx);
    sum = team_sum(s, s_redf, g, T);
  }

  // ---- 2./3. chunks of R ranks ----
  const int slice = s0 + g;
  const size_t out0 = (size_t)blockIdx.y * k * ns;
  const uint8_t* cb = code != nullptr ? code + blockIdx.y * vol : nullptr;
  unsigned long long hi = ~0ull;          // keys of the ranks already written are >= hi
  for (int r0 = 0; r0 < k; r0 += R) {
    const int cnt = min(R, k - r0);
    // radix select: the key of rank r0 + cnt (1-based), or a prefix below it and above every lower rank
    if (lt == 0) {
      s_prefix[g] = 0;
      s_rem[g] = r0 + cnt;
      s_done[g] = 0;
    }
    for (int shift = 40; shift >= 0; shift -= 8) {
      for (int d = lt; d < 256; d += T) hist[g][d] = 0;
      __syncthreads();
      const unsigned long long pre = s_prefix[g];
      if (!s_done[g]) {
        for (int base = 0; base < N; base += T) {
          const int i = base + lt;
          int digit = -1;
          if (i < N) {
            const unsigned long long c = topk_key(kv[i], i);
            if ((c >> (shift + 8)) == (pre >> (shift + 8))) digit = (int)((c >> shift) & 255);
          }
          const unsigned peers = __match_any_sync(0xffffffffu, digit);
          if (digit >= 0 && (threadIdx.x & 31) == __ffs(peers) - 1) atomicAdd(&hist[g][digit], __popc(peers));
        }
      }
      __syncthreads();
      if (lt < 32 && !s_done[g]) {        // lane l holds bins 255 - 8l .. 248 - 8l, counted from the top
        unsigned tot = 0;
#pragma unroll
        for (int j = 0; j < 8; ++j) tot += hist[g][255 - 8 * lt - j];
        unsigned incl = tot;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
          const unsigned v = __shfl_up_sync(0xffffffffu, incl, o);
          if (lt >= o) incl += v;
        }
        const unsigned rem = s_rem[g];
        const int L = __ffs(__ballot_sync(0xffffffffu, incl >= rem)) - 1;
        if (lt == L) {
          unsigned before = incl - tot;
          for (int j = 0; j < 8; ++j) {
            const unsigned c = hist[g][255 - 8 * L - j];
            if (before + c >= rem) {
              s_prefix[g] = pre | ((unsigned long long)(255 - 8 * L - j) << shift);
              s_rem[g] = rem - before;
              s_done[g] = before + c == rem;        // the bin holds exactly the ranks still needed
              break;
            }
            before += c;
          }
        }
      }
      if (__syncthreads_and(s_done[g])) break;
    }
    const unsigned long long lo = s_prefix[g];

    // compact the chunk's keys (exactly cnt of them) and sort them, descending
    int n2 = 1;
    while (n2 < cnt) n2 <<= 1;
    for (int p = lt; p < n2; p += T) buf[p] = 0;     // padding sorts last: every real key is > 0
    if (lt == 0) s_ctr[g] = 0;
    __syncthreads();
    for (int i = lt; i < N; i += T) {
      const unsigned long long c = topk_key(kv[i], i);
      if (c >= lo && c < hi) buf[atomicAdd(&s_ctr[g], 1u)] = c;
    }
    __syncthreads();
    for (int size = 2; size <= n2; size <<= 1) {
      for (int j = size >> 1; j > 0; j >>= 1) {
        for (int q = lt; q < (n2 >> 1); q += T) {
          const int i = ((q & ~(j - 1)) << 1) | (q & (j - 1));
          const unsigned long long a = buf[i], b = buf[i + j];
          if ((a < b) == ((i & size) == 0)) {
            buf[i] = b;
            buf[i + j] = a;
          }
        }
        __syncthreads();
      }
    }

    if (slice < ns) {
      for (int p = lt; p < cnt; p += T) {
        const unsigned long long c = buf[p];
        const int idx = 0xffff - (int)(c & 0xffff);
        const float v = ord2f((unsigned)(c >> 16));
        const int a = INVERT ? slice : idx, b = INVERT ? idx : slice;
        int iA = a / wA, jA = a - iA * wA, iB = b / wB, jB = b - iB * wB;
        if (cb != nullptr) {             // code = ((di * ks + dj) * ks + dk) * ks + dl, as delta_pack_kernel packs it
          int cc = cb[(size_t)a * nB + b];
          const int dl = cc % ks; cc /= ks;
          const int dk = cc % ks; cc /= ks;
          const int dj = cc % ks; cc /= ks;
          iA = iA * ks + cc; jA = jA * ks + dj; iB = iB * ks + dk; jB = jB * ks + dl;
        }
        const int rank = r0 + p;
        const size_t o = out0 + (INVERT ? (size_t)slice * k + rank : (size_t)rank * ns + slice);
        jA_out[o] = jA;
        iA_out[o] = iA;
        jB_out[o] = jB;
        iB_out[o] = iB;
        sc_out[o] = do_softmax ? __fdiv_rn(expf(v - mx), sum) : v;
      }
    }
    hi = lo;
    __syncthreads();                      // buf and the select state are reused by the next chunk
  }
}

// -> G slices per CTA, R ranks per chunk, dynamic shared memory; -1 when n_slice or k is out of range
int corr_topk_config(int n_slice, int k, int* G, int* R, size_t* smem) {
  if (n_slice < 1 || n_slice > kTopkMaxSlice || k < 1 || k > n_slice) return -1;
  const int g = n_slice <= 4096 ? 8 : n_slice <= 8192 ? 4 : n_slice <= 16384 ? 2 : 1;
  int r = 1;
  while (r < k && r < 8192 / g) r <<= 1;
  *G = g;
  *R = r;
  *smem = (size_t)g * r * 8 + (size_t)g * (n_slice + 1) * 4;
  return 0;
}

}  // namespace

int launch_corr_topk(const float* corr, const uint8_t* code, int b, int hA, int wA, int hB, int wB, int k, int ks,
                     int do_softmax, int invert, long long* jA, long long* iA, long long* jB, long long* iB,
                     float* score, cudaStream_t st) {
  const int nA = hA * wA, nB = hB * wB;
  const int n_slice = invert ? nB : nA, ns = invert ? nA : nB;
  int G, R;
  size_t smem;
  P2P_REQUIRE(corr_topk_config(n_slice, k, &G, &R, &smem) == 0, "slice length or topk out of range");
  const dim3 grid(cdiv(ns, G), b);
  if (invert) {
    P2P_ENSURE_SMEM(corr_topk_kernel<true>, smem);
    corr_topk_kernel<true><<<grid, kTopkThreads, smem, st>>>(corr, code, nA, nB, wA, wB, G, R, k, ks, do_softmax, jA,
                                                              iA, jB, iB, score);
  } else {
    P2P_ENSURE_SMEM(corr_topk_kernel<false>, smem);
    corr_topk_kernel<false><<<grid, kTopkThreads, smem, st>>>(corr, code, nA, nB, wA, wB, G, R, k, ks, do_softmax, jA,
                                                               iA, jB, iB, score);
  }
  P2P_LAUNCH_OK();
  return 0;
}

}  // namespace p2p
