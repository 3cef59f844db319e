// SuperGlue's log-domain optimal transport and mutual match extraction (semantics in include/p2p_b200.h,
// p2p_sg_sinkhorn; the float64 restatement in oracle/superglue_oracle.py).
//
//   one cooperative launch per call, cooperative_groups grid syncs between its phases:
//     0  tiled transpose of the scores Z [b][n][m] into the scratch copy Zt [b][m][n]; u = v = 0
//     1  per iteration, two row passes: u_i from the rows of Z and v, then v_j from the rows of Zt and u.  The dustbin
//        row and column are virtual (alpha); the couplings are never materialised
//     2  the last pass: log_assign (when asked for), each row's max / argmax over Z and each column's over Zt, from
//        the same fp32 expression ((C + u_i) + v_j) - norm, so both see the bits log_assign holds
//     3  mutual test, threshold, matches and scores
//   One warp owns one output row of a pass: an online log-sum-exp over the row in a fixed lane-strided order (chunks of
//   kChunk elements per lane), combined across lanes by a fixed xor butterfly.  No atomics and no cross-warp partial
//   sums, so every u_i / v_j depends only on its own row: results are bit-identical for any grid size and a pair gives
//   the same bits alone or inside a batch.
#include <cooperative_groups.h>

#include <algorithm>
#include <cmath>

#include "common.cuh"
#include "kernels.h"

namespace cg = cooperative_groups;

namespace p2p {
namespace {

constexpr int kSgThreads = 256;
constexpr int kSgWarps = kSgThreads / 32;
constexpr int kChunk = 8;        // elements per lane per step of a row pass: a warp covers 256 columns per step
constexpr int kTile = 32;        // transpose tile

struct SgArgs {
  const float* Z;      // [B][n][m]
  float* Zt;           // [B][m][n] scratch
  const float* alpha;  // device scalar
  float* u;            // [B][n + 1]
  float* v;            // [B][m + 1]
  float* rmax;         // [B][n] row maxima (the decisions need no column maxima)
  int* rarg;           // [B][n]
  int* carg;           // [B][m]
  float* la;           // [B][n + 1][m + 1] or null
  int* m0;             // [B][n] or null
  int* m1;             // [B][m] or null
  float* s0;           // [B][n] or null
  float* s1;           // [B][m] or null
  int B, n, m, iters;
  float norm, lmu_bin, lnu_bin, thr;   // norm = -log(n + m), log(m) + norm, log(n) + norm (rounded from double)
};

// max that returns NaN when either input is NaN (fmaxf returns the other input)
__device__ __forceinline__ float fmax_nan(float a, float b) {
  float d;
  asm("max.NaN.f32 %0, %1, %2;" : "=f"(d) : "f"(a), "f"(b));
  return d;
}

// u_out[r] = (i < rows ? lnorm : lbin) - LSE_j(c_ij + v_j), j = 0 .. cols, for every row r = (b, i) of a pass over
// M [B][rows][cols]; c_ij = M[b][i][j] for i < rows and j < cols, alpha otherwise (the dustbin row / column).
__device__ __forceinline__ void lse_pass(const float* __restrict__ M, int B, int rows, int cols, float alpha,
                                         const float* vin, float* uout, float lnorm, float lbin, int gw, int nw,
                                         int lane) {
  const int total = B * (rows + 1);
  for (int r = gw; r < total; r += nw) {
    const int b = r / (rows + 1), i = r - b * (rows + 1);
    const float* row = i < rows ? M + ((size_t)b * rows + i) * cols : nullptr;
    const float* vb = vin + (size_t)b * (cols + 1);
    float mx = -INFINITY, s = 0.f;
    for (int base = 0; base <= cols; base += 32 * kChunk) {
      float x[kChunk];
      float cm = -INFINITY;
#pragma unroll
      for (int k = 0; k < kChunk; ++k) {
        const int j = base + k * 32 + lane;
        const float c = (row != nullptr && j < cols) ? __ldcg(row + j) : alpha;
        x[k] = j <= cols ? c + vb[j] : -INFINITY;
        cm = fmax_nan(cm, x[k]);                      // a NaN term makes cm, then s, NaN, as in float64
      }
      if (cm == -INFINITY) continue;                  // past the row's end, or masked (-inf)
      if (cm > mx) {
        s *= expf(mx - cm);                           // expf(-inf) = 0 on the first chunk
        mx = cm;
      }
      float cs = 0.f;
#pragma unroll
      for (int k = 0; k < kChunk; ++k) cs += expf(x[k] - mx);
      s += cs;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float om = __shfl_xor_sync(0xffffffffu, mx, o), os = __shfl_xor_sync(0xffffffffu, s, o);
      const float M2 = fmaxf(mx, om);
      s = M2 == -INFINITY ? s + os : s * expf(mx - M2) + os * expf(om - M2);   // s + os: 0, or NaN kept
      mx = M2;
    }
    if (lane == 0) uout[r] = (i < rows ? lnorm : lbin) - (mx + logf(s));
  }
}

// Running (value, index) max in np.argmax's order: NaN above +inf above every number above -inf, ties (NaN with NaN
// included) to the lowest index.
__device__ __forceinline__ void arg_combine(float& bv, int& bi, float ov, int oi) {
  const bool on = ov != ov, bn = bv != bv;
  if (on != bn ? on : (ov > bv || (!(ov < bv) && oi < bi))) {
    bv = ov;
    bi = oi;
  }
}

__device__ __forceinline__ void warp_argmax(float& bv, int& bi) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    arg_combine(bv, bi, ov, oi);
  }
}

__global__ void __launch_bounds__(kSgThreads) sg_sinkhorn_kernel(SgArgs a) {
  cg::grid_group grid = cg::this_grid();
  const int B = a.B, n = a.n, m = a.m;
  const float alpha = *a.alpha;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int gw = blockIdx.x * kSgWarps + warp, nw = gridDim.x * kSgWarps;
  const long long gt = (long long)blockIdx.x * kSgThreads + threadIdx.x, nt = (long long)gridDim.x * kSgThreads;

  // ---- phase 0: Zt = Z^T per pair, u = v = 0
  {
    __shared__ float tile[kTile][kTile + 1];
    const int tn = (n + kTile - 1) / kTile, tm = (m + kTile - 1) / kTile;
    const long long tiles = (long long)B * tn * tm;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    for (long long t = blockIdx.x; t < tiles; t += gridDim.x) {
      const int b = (int)(t / ((long long)tn * tm));
      const int q = (int)(t - (long long)b * tn * tm);
      const int i0 = (q / tm) * kTile, j0 = (q % tm) * kTile;
      const float* src = a.Z + (size_t)b * n * m;
      for (int y = ty; y < kTile; y += kSgWarps)
        if (i0 + y < n && j0 + tx < m) tile[y][tx] = src[(size_t)(i0 + y) * m + j0 + tx];
      __syncthreads();
      float* dst = a.Zt + (size_t)b * n * m;
      for (int y = ty; y < kTile; y += kSgWarps)
        if (j0 + y < m && i0 + tx < n) dst[(size_t)(j0 + y) * n + i0 + tx] = tile[tx][y];
      __syncthreads();
    }
    for (long long k = gt; k < (long long)B * (n + 1); k += nt) a.u[k] = 0.f;
    for (long long k = gt; k < (long long)B * (m + 1); k += nt) a.v[k] = 0.f;
  }
  grid.sync();

  // ---- phase 1: Sinkhorn iterations
  for (int it = 0; it < a.iters; ++it) {
    lse_pass(a.Z, B, n, m, alpha, a.v, a.u, a.norm, a.lmu_bin, gw, nw, lane);
    grid.sync();
    lse_pass(a.Zt, B, m, n, alpha, a.u, a.v, a.norm, a.lnu_bin, gw, nw, lane);
    grid.sync();
  }

  // ---- phase 2: log_assign, row maxima over Z, column maxima over Zt
  const float norm = a.norm;
  for (int r = gw; r < B * (n + 1) + B * m; r += nw) {
    if (r < B * (n + 1)) {
      const int b = r / (n + 1), i = r - b * (n + 1);
      const float ui = a.u[r];
      const float* vb = a.v + (size_t)b * (m + 1);
      float* out = a.la != nullptr ? a.la + (size_t)r * (m + 1) : nullptr;
      if (i == n) {   // the dustbin row: log_assign only
        if (out != nullptr)
          for (int j = lane; j <= m; j += 32) out[j] = ((alpha + ui) + vb[j]) - norm;
        continue;
      }
      const float* row = a.Z + ((size_t)b * n + i) * m;
      // every lane starts as if on a -inf at a real column (its first, or 0 past m): the first element replaces it
      // unless it is -inf too, so the index is in [0, m) for any values, and for any compare in arg_combine
      float bv = -INFINITY;
      int bi = lane < m ? lane : 0;
      for (int j = lane; j < m; j += 32) {
        const float z = ((__ldcg(row + j) + ui) + vb[j]) - norm;
        if (out != nullptr) out[j] = z;
        if (z > bv || (z != z && bv == bv)) {         // j rises: the lane keeps its first maximum, or first NaN
          bv = z;
          bi = j;
        }
      }
      if (out != nullptr && lane == 0) out[m] = ((alpha + ui) + vb[m]) - norm;
      warp_argmax(bv, bi);
      if (lane == 0) {
        a.rmax[(size_t)b * n + i] = bv;
        a.rarg[(size_t)b * n + i] = bi;
      }
    } else {
      const int c = r - B * (n + 1);
      const int b = c / m, j = c - b * m;
      const float vj = a.v[(size_t)b * (m + 1) + j];
      const float* ub = a.u + (size_t)b * (n + 1);
      const float* col = a.Zt + ((size_t)b * m + j) * n;
      float bv = -INFINITY;                           // as for rows: the index is in [0, n) for any values
      int bi = lane < n ? lane : 0;
      for (int i = lane; i < n; i += 32) {
        const float z = ((__ldcg(col + i) + ub[i]) + vj) - norm;
        if (z > bv || (z != z && bv == bv)) {
          bv = z;
          bi = i;
        }
      }
      warp_argmax(bv, bi);
      if (lane == 0) a.carg[c] = bi;
    }
  }
  grid.sync();

  // ---- phase 3: mutual test, threshold, outputs
  for (long long k = gt; k < (long long)B * n + (long long)B * m; k += nt) {
    if (k < (long long)B * n) {
      const int b = (int)(k / n);
      const int j = a.rarg[k];
      const bool mutual = a.carg[(size_t)b * m + j] == (int)(k - (long long)b * n);
      const float sc = mutual ? expf(a.rmax[k]) : 0.f;
      if (a.m0 != nullptr) a.m0[k] = mutual && sc > a.thr ? j : -1;
      if (a.s0 != nullptr) a.s0[k] = sc;
    } else {
      const long long c = k - (long long)B * n;
      const int b = (int)(c / m);
      const int i = a.carg[c];
      const size_t ri = (size_t)b * n + i;
      const bool mutual = a.rarg[ri] == (int)(c - (long long)b * m);
      const float sc = mutual ? expf(a.rmax[ri]) : 0.f;   // mscores0 of row i, which is mutual when column j is
      if (a.m1 != nullptr) a.m1[c] = mutual && sc > a.thr ? i : -1;
      if (a.s1 != nullptr) a.s1[c] = sc;
    }
  }
}

}  // namespace

size_t sg_sinkhorn_scratch_bytes(int B, int n, int m) {
  const size_t nm = (size_t)B * n * m, pn = (size_t)B * (n + 1), pm = (size_t)B * (m + 1);
  return align_up(nm * 4 + 272, 256) + align_up(pn * 4 + 272, 256) + align_up(pm * 4 + 272, 256) +
         2 * align_up((size_t)B * n * 4 + 272, 256) + align_up((size_t)B * m * 4 + 272, 256);
}

int launch_sg_sinkhorn(Arena& ar, const float* scores, int B, int n, int m, const float* alpha, int iters, float thr,
                       float* log_assign, int* matches0, int* matches1, float* mscores0, float* mscores1, int sms,
                       cudaStream_t st) {
  const size_t need = sg_sinkhorn_scratch_bytes(B, n, m);
  if (int rc = ar.reserve(need + 1024)) return rc;
  Carve cv{(char*)ar.take(need)};
  P2P_REQUIRE(cv.p != nullptr, "scratch carve failed");
  SgArgs a;
  a.Z = scores;
  a.Zt = cv.take<float>((size_t)B * n * m);
  a.alpha = alpha;
  a.u = cv.take<float>((size_t)B * (n + 1));
  a.v = cv.take<float>((size_t)B * (m + 1));
  a.rmax = cv.take<float>((size_t)B * n);
  a.rarg = cv.take<int>((size_t)B * n);
  a.carg = cv.take<int>((size_t)B * m);
  a.la = log_assign;
  a.m0 = matches0;
  a.m1 = matches1;
  a.s0 = mscores0;
  a.s1 = mscores1;
  a.B = B;
  a.n = n;
  a.m = m;
  a.iters = iters;
  const double norm = -std::log((double)n + (double)m);
  a.norm = (float)norm;
  a.lmu_bin = (float)(std::log((double)m) + norm);
  a.lnu_bin = (float)(std::log((double)n) + norm);
  a.thr = thr;

  int per_sm = 0;
  P2P_CUDA_OK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, sg_sinkhorn_kernel, kSgThreads, 0));
  P2P_REQUIRE(per_sm >= 1, "sg_sinkhorn_kernel does not fit on an SM");
  // work: the widest phase, in blocks (rows of a pass or of the last pass per warp, transpose tiles per block)
  const long long rows = std::max((long long)B * (n + 1) + (long long)B * m, (long long)B * (m + 1));
  const long long tiles = (long long)B * cdiv(n, kTile) * cdiv(m, kTile);
  const long long work = std::max((rows + kSgWarps - 1) / kSgWarps, tiles);
  const int grid = (int)std::max(1ll, std::min((long long)per_sm * sms, work));
  void* args[] = {&a};
  P2P_CUDA_OK(cudaLaunchCooperativeKernel((const void*)sg_sinkhorn_kernel, dim3(grid), dim3(kSgThreads), args, 0, st));
  P2P_LAUNCH_OK();
  return 0;
}

}  // namespace p2p
