// Coarse stage: L2-normalise -> 4D correlation (+4D max-pool) -> MutualMatching -> symmetric
// 4D neighbourhood-consensus conv -> MutualMatching -> softmax/argmax proposals -> unique/mutual.
//
// Reference semantics (file:line relative to the reference repo):
//   L2Normalize            networks/modules.py:6
//   FeatCorrelation        networks/modules.py:36-53
//   maxpool4d              networks/modules.py:11-34
//   MutualMatching         networks/ncn/model.py:157-176
//   NeighConsensus/Conv4d  networks/ncn/model.py:124-155, networks/ncn/conv4d.py:12-74
//   corr_to_matches        networks/ncn/extract_ncmatches.py:6-94
//   cal_coarse_matches     networks/patch2pix.py:340-375
//   filter_coarse (unique) networks/utils.py:38-50
//
// All arithmetic here is fp32 FMA on the CUDA cores: "proposal indices bit-exact" needs
// fp32-grade correlation / NC scores (SURVEY.md s0, H1).  The tensor-core correlation lives in
// umma_gemm.cuh; this file keeps the HBM-bound scans and the fp32 NC convolution.
#include "kernels.h"

namespace p2p {

// ------------------------------------------------------------------------------------------------
// K1: L2 normalise over channels and (for ksize 2) permute positions into pooling-window order:
// out[c][cell*4 + m], m = di*2+dj, so that the 4 members of a 2x2 window are adjacent.
// ------------------------------------------------------------------------------------------------
template <int KS>
__global__ void __launch_bounds__(256) l2norm_perm_kernel(const float* __restrict__ in, float* __restrict__ out,
                                                         int C, int h, int w) {
  const int n = h * w;
  const int q = blockIdx.x * blockDim.x + threadIdx.x;  // output index
  if (q >= n) return;
  int pos;
  if (KS == 2) {
    const int wp = w >> 1;
    const int cell = q >> 2, m = q & 3;
    const int pi = cell / wp, pj = cell - pi * wp;
    pos = (2 * pi + (m >> 1)) * w + 2 * pj + (m & 1);
  } else {
    pos = q;
  }
  float s = 0.f;
  for (int c = 0; c < C; ++c) {
    const float v = __ldg(in + (size_t)c * n + pos);
    s = fmaf(v, v, s);
  }
  const float d = sqrtf(s + 1e-6f);
  for (int c = 0; c < C; ++c) out[(size_t)c * n + q] = __ldg(in + (size_t)c * n + pos) / d;
}

// ------------------------------------------------------------------------------------------------
// K2+K3 (CUDA-core variant): corr[m][n] = sum_c A[c][m] B[c][n] with the 2^4 max-pool and the
// argmax code fused into the epilogue.  Each thread owns a 4x4 micro-tile which, thanks to the
// window-order permutation above, is exactly one 4D pooling window.
// code = ((di*2+dj)*2+dk)*2+dl with ties resolved to the lowest code (torch.max semantics).
// ------------------------------------------------------------------------------------------------
template <int KS>
__global__ void __launch_bounds__(256) corr_pool_kernel(const float* __restrict__ fa, const float* __restrict__ fb,
                                                       int C, int n1, int n2, float* __restrict__ out,
                                                       uint8_t* __restrict__ code) {
  constexpr int KC = 16;
  __shared__ __align__(16) float As[KC][64];
  __shared__ __align__(16) float Bs[KC][64];
  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;
  const int a0 = blockIdx.y * 64, b0 = blockIdx.x * 64;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  for (int k0 = 0; k0 < C; k0 += KC) {
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const int idx = tid + r * 256;
      const int kk = idx >> 6, q = idx & 63;
      const bool kin = (k0 + kk) < C;
      As[kk][q] = (kin && a0 + q < n1) ? __ldg(fa + (size_t)(k0 + kk) * n1 + a0 + q) : 0.f;
      Bs[kk][q] = (kin && b0 + q < n2) ? __ldg(fb + (size_t)(k0 + kk) * n2 + b0 + q) : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < KC; ++kk) {
      const float4 a = *reinterpret_cast<const float4*>(&As[kk][ty * 4]);
      const float4 b = *reinterpret_cast<const float4*>(&Bs[kk][tx * 4]);
      const float av[4] = {a.x, a.y, a.z, a.w};
      const float bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    __syncthreads();
  }
  if (KS == 2) {
    const int np1 = n1 >> 2, np2 = n2 >> 2;
    const int ca = (a0 >> 2) + ty, cb = (b0 >> 2) + tx;
    if (ca < np1 && cb < np2) {
      float best = acc[0][0];
      int bi = 0;
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j)
          if (acc[i][j] > best) {
            best = acc[i][j];
            bi = i * 4 + j;
          }
      out[(size_t)ca * np2 + cb] = best;
      code[(size_t)ca * np2 + cb] = (uint8_t)bi;
    }
  } else {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int row = a0 + ty * 4 + i;
      if (row >= n1) continue;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int col = b0 + tx * 4 + j;
        if (col < n2) out[(size_t)row * n2 + col] = acc[i][j];
      }
    }
  }
}

// K-major fp16 hi/lo output for the tensor-core correlation.  Block = 32 consecutive output positions x all channels:
// coalesced reads along the positions (NCHW input), transposed through shared memory, 64-byte row segments out.
// Both images in one launch (blockIdx.y).
struct L2NormArgs {
  const float* in[2];
  __half* hi[2];
  __half* lo[2];
  int h[2], w[2];
};

template <int KS>
__global__ void __launch_bounds__(256) l2norm_perm_kmajor_kernel(const __grid_constant__ L2NormArgs a, int C) {
  extern __shared__ float tile[];      // [C][33]
  __shared__ float part[8][32];
  __shared__ float dinv[32];
  const int im = blockIdx.y;
  const int h = a.h[im], w = a.w[im], n = h * w;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int q0 = blockIdx.x * 32;
  if (q0 >= n) return;
  const int q = q0 + lane;
  int pos = 0;
  if (q < n) {
    if (KS == 2) {
      const int wp = w >> 1;
      const int cell = q >> 2, m = q & 3;
      const int pi = cell / wp, pj = cell - pi * wp;
      pos = (2 * pi + (m >> 1)) * w + 2 * pj + (m & 1);
    } else {
      pos = q;
    }
  }
  const float* in = a.in[im];
  float s = 0.f;
  for (int c = wid; c < C; c += 8) {
    const float v = q < n ? __ldg(in + (size_t)c * n + pos) : 0.f;
    tile[c * 33 + lane] = v;
    s = fmaf(v, v, s);
  }
  part[wid][lane] = s;
  __syncthreads();
  if (wid == 0) {
    float t = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) t += part[i][lane];
    dinv[lane] = sqrtf(t + 1e-6f);
  }
  __syncthreads();
  __half* hi = a.hi[im];
  __half* lo = a.lo[im];
  for (int i = threadIdx.x; i < 32 * (C / 2); i += 256) {
    const int p = i / (C / 2), c = (i - p * (C / 2)) * 2;
    if (q0 + p >= n) continue;
    const float d = dinv[p];
    const float v0 = __fdiv_rn(tile[c * 33 + p], d) * kActScale, v1 = __fdiv_rn(tile[(c + 1) * 33 + p], d) * kActScale;
    const __half2 hh = __floats2half2_rn(v0, v1);
    *reinterpret_cast<__half2*>(hi + (size_t)(q0 + p) * C + c) = hh;
    if (lo != nullptr) {
      const float2 f = __half22float2(hh);
      *reinterpret_cast<__half2*>(lo + (size_t)(q0 + p) * C + c) = __floats2half2_rn(v0 - f.x, v1 - f.y);
    }
  }
}

int launch_l2norm_perm_kmajor_pair(const float* in1, const float* in2, __half* hi1, __half* lo1, __half* hi2, __half* lo2,
                                   int C, int h1, int w1, int h2, int w2, int ksize, cudaStream_t st) {
  P2P_REQUIRE(C % 2 == 0 && C <= 1024, "l2norm: channel count must be even and at most 1024");
  L2NormArgs a;
  a.in[0] = in1; a.in[1] = in2;
  a.hi[0] = hi1; a.hi[1] = hi2;
  a.lo[0] = lo1; a.lo[1] = lo2;
  a.h[0] = h1; a.w[0] = w1; a.h[1] = h2; a.w[1] = w2;
  const int nmax = h1 * w1 > h2 * w2 ? h1 * w1 : h2 * w2;
  dim3 grid(cdiv(nmax, 32), 2);
  const size_t smem = sizeof(float) * C * 33;
  if (ksize == 2) {
    P2P_ENSURE_SMEM(l2norm_perm_kmajor_kernel<2>, smem);
    l2norm_perm_kmajor_kernel<2><<<grid, 256, smem, st>>>(a, C);
  } else {
    P2P_ENSURE_SMEM(l2norm_perm_kmajor_kernel<1>, smem);
    l2norm_perm_kmajor_kernel<1><<<grid, 256, smem, st>>>(a, C);
  }
  P2P_LAUNCH_OK();
  return 0;
}

// Same, for a channels-last fp16 layer-3 map [n][C] (the fp16 / channels_last backbone of the end-to-end path):
// the input is already K-major, so this is a row-wise normalise + hi/lo split; one warp per output position.
template <int KS>
__global__ void __launch_bounds__(256) l2norm_perm_kmajor_nhwc16_kernel(const __grid_constant__ L2NormArgs a, int C) {
  const int im = blockIdx.y;
  const int h = a.h[im], w = a.w[im], n = h * w;
  const int lane = threadIdx.x & 31;
  const int q = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (q >= n) return;
  int pos;
  if (KS == 2) {
    const int wp = w >> 1;
    const int cell = q >> 2, m = q & 3;
    const int pi = cell / wp, pj = cell - pi * wp;
    pos = (2 * pi + (m >> 1)) * w + 2 * pj + (m & 1);
  } else {
    pos = q;
  }
  const __half* in = reinterpret_cast<const __half*>(a.in[im]) + (size_t)pos * C;
  float s = 0.f;
  for (int c = lane * 8; c < C; c += 256) {
    const uint4 v = __ldg(reinterpret_cast<const uint4*>(in + c));
    const __half2* h2 = reinterpret_cast<const __half2*>(&v);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float2 f = __half22float2(h2[i]);
      s = fmaf(f.x, f.x, s);
      s = fmaf(f.y, f.y, s);
    }
  }
  s = warp_sum(s);
  const float d = sqrtf(s + 1e-6f);
  __half* hi = a.hi[im] + (size_t)q * C;
  __half* lo = a.lo[im] != nullptr ? a.lo[im] + (size_t)q * C : nullptr;
  for (int c = lane * 8; c < C; c += 256) {
    const uint4 v = __ldg(reinterpret_cast<const uint4*>(in + c));
    const __half2* h2 = reinterpret_cast<const __half2*>(&v);
    __align__(16) __half2 oh[4];
    __align__(16) __half2 ol[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float2 f = __half22float2(h2[i]);
      const float v0 = __fdiv_rn(f.x, d) * kActScale, v1 = __fdiv_rn(f.y, d) * kActScale;
      oh[i] = __floats2half2_rn(v0, v1);
      const float2 g = __half22float2(oh[i]);
      ol[i] = __floats2half2_rn(v0 - g.x, v1 - g.y);
    }
    *reinterpret_cast<uint4*>(hi + c) = *reinterpret_cast<const uint4*>(oh);
    if (lo != nullptr) *reinterpret_cast<uint4*>(lo + c) = *reinterpret_cast<const uint4*>(ol);
  }
}

int launch_l2norm_perm_kmajor_pair_nhwc16(const __half* in1, const __half* in2, __half* hi1, __half* lo1, __half* hi2, __half* lo2,
                                          int C, int h1, int w1, int h2, int w2, int ksize, cudaStream_t st) {
  P2P_REQUIRE(C % 8 == 0, "l2norm (channels-last fp16): channel count must be a multiple of 8");
  L2NormArgs a;
  a.in[0] = reinterpret_cast<const float*>(in1); a.in[1] = reinterpret_cast<const float*>(in2);
  a.hi[0] = hi1; a.hi[1] = hi2;
  a.lo[0] = lo1; a.lo[1] = lo2;
  a.h[0] = h1; a.w[0] = w1; a.h[1] = h2; a.w[1] = w2;
  const int nmax = h1 * w1 > h2 * w2 ? h1 * w1 : h2 * w2;
  dim3 grid(cdiv(nmax, 8), 2);
  if (ksize == 2) l2norm_perm_kmajor_nhwc16_kernel<2><<<grid, 256, 0, st>>>(a, C);
  else l2norm_perm_kmajor_nhwc16_kernel<1><<<grid, 256, 0, st>>>(a, C);
  P2P_LAUNCH_OK();
  return 0;
}

__global__ void split_rows_kernel(const float* __restrict__ in, __half* __restrict__ hi, __half* __restrict__ lo,
                                  size_t n, float scale) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float v = in[i] * scale;
  const __half hh = __float2half_rn(v);
  hi[i] = hh;
  if (lo != nullptr) lo[i] = __float2half_rn(v - __half2float(hh));
}

int launch_split_rows(const float* in, __half* hi, __half* lo, size_t n, float scale, cudaStream_t st) {
  split_rows_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(in, hi, lo, n, scale);
  P2P_LAUNCH_OK();
  return 0;
}

__global__ void delta_pack_kernel(const long long* di, const long long* dj, const long long* dk, const long long* dl,
                                  size_t n, int ks, uint8_t* code) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  code[i] = (uint8_t)(((di[i] * ks + dj[i]) * ks + dk[i]) * ks + dl[i]);
}

int launch_delta_pack(const long long* di, const long long* dj, const long long* dk, const long long* dl, size_t n,
                      int ks, uint8_t* code, cudaStream_t st) {
  delta_pack_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(di, dj, dk, dl, n, ks, code);
  P2P_LAUNCH_OK();
  return 0;
}

int launch_l2norm_perm(const float* in, float* out, int C, int h, int w, int ksize, cudaStream_t st) {
  const int n = h * w;
  if (ksize == 2)
    l2norm_perm_kernel<2><<<cdiv(n, 256), 256, 0, st>>>(in, out, C, h, w);
  else
    l2norm_perm_kernel<1><<<cdiv(n, 256), 256, 0, st>>>(in, out, C, h, w);
  P2P_LAUNCH_OK();
  return 0;
}

int launch_corr_pool_simt(const float* fa, const float* fb, int C, int n1, int n2, int ksize, float* out,
                          uint8_t* code, cudaStream_t st) {
  dim3 grid(cdiv(n2, 64), cdiv(n1, 64));
  if (ksize == 2)
    corr_pool_kernel<2><<<grid, 256, 0, st>>>(fa, fb, C, n1, n2, out, code);
  else
    corr_pool_kernel<1><<<grid, 256, 0, st>>>(fa, fb, C, n1, n2, out, code);
  P2P_LAUNCH_OK();
  return 0;
}

// Expand the packed argmax code into the reference's four int64 delta tensors.
__global__ void delta_unpack_kernel(const uint8_t* __restrict__ code, size_t n, int ks, long long* di, long long* dj,
                                    long long* dk, long long* dl) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int c = code[i];
  const int l = c % ks;
  c /= ks;
  const int k = c % ks;
  c /= ks;
  const int j = c % ks;
  c /= ks;
  di[i] = c;
  dj[i] = j;
  dk[i] = k;
  dl[i] = l;
}

int launch_delta_unpack(const uint8_t* code, size_t n, int ks, long long* di, long long* dj, long long* dk,
                        long long* dl, cudaStream_t st) {
  delta_unpack_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(code, n, ks, di, dj, dk, dl);
  P2P_LAUNCH_OK();
  return 0;
}

// ------------------------------------------------------------------------------------------------
// K4: MutualMatching.  rowmax[a] = max_b x[a][b] (max over B for a fixed A cell),
// colmax[b] = max_a x[a][b]; out = x * ((x/(rowmax+eps)) * (x/(colmax+eps))).
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) rowcolmax_kernel(const float* __restrict__ x, int nA, int nB,
                                                       float* __restrict__ rowmax, unsigned int* __restrict__ colmax) {
  constexpr int R = 8;
  __shared__ float red[8][R];
  const int r0 = blockIdx.x * R;
  float rm[R];
#pragma unroll
  for (int r = 0; r < R; ++r) rm[r] = -INFINITY;
  for (int col = threadIdx.x; col < nB; col += 256) {
    float cm = -INFINITY;
#pragma unroll
    for (int r = 0; r < R; ++r) {
      if (r0 + r < nA) {
        const float v = x[(size_t)(r0 + r) * nB + col];
        rm[r] = fmaxf(rm[r], v);
        cm = fmaxf(cm, v);
      }
    }
    atomicMax(colmax + col, f2ord(cm));
  }
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
  for (int r = 0; r < R; ++r) {
    const float v = warp_max(rm[r]);
    if (lane == 0) red[wid][r] = v;
  }
  __syncthreads();
  if (threadIdx.x < R && r0 + threadIdx.x < nA) {
    float v = red[0][threadIdx.x];
#pragma unroll
    for (int wv = 1; wv < 8; ++wv) v = fmaxf(v, red[wv][threadIdx.x]);
    rowmax[r0 + threadIdx.x] = v;
  }
}

__global__ void __launch_bounds__(256) mutual_apply_kernel(const float* __restrict__ x, int nA, int nB,
                                                          const float* __restrict__ rowmax,
                                                          const unsigned int* __restrict__ colmax,
                                                          float* __restrict__ out, unsigned int* __restrict__ absmax) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  float o = 0.f;
  if (i < (size_t)nA * nB) {
    const int a = (int)(i / nB), b = (int)(i - (size_t)a * nB);
    const float v = x[i];
    const float ra = __fdiv_rn(v, rowmax[a] + 1e-5f);
    const float rb = __fdiv_rn(v, ord2f(colmax[b]) + 1e-5f);
    o = __fmul_rn(v, __fmul_rn(ra, rb));
    out[i] = o;
  }
  if (absmax != nullptr) {      // block-uniform: one atomic per block (non-negative floats order like their bits)
    __shared__ float s_m[8];
    const float m = warp_max(fabsf(o));
    if ((threadIdx.x & 31) == 0) s_m[threadIdx.x >> 5] = m;
    __syncthreads();
    if (threadIdx.x == 0) {
      float t = s_m[0];
#pragma unroll
      for (int i = 1; i < 8; ++i) t = fmaxf(t, s_m[i]);
      if (t > 0.f) atomicMax(absmax, __float_as_uint(t));
    }
  }
}

int launch_mutual_apply(const float* x, int nA, int nB, const float* rowmax, const unsigned int* colmax, float* out,
                        unsigned int* absmax, cudaStream_t st) {
  if (absmax != nullptr) P2P_CUDA_OK(cudaMemsetAsync(absmax, 0, sizeof(unsigned int), st));
  const size_t n = (size_t)nA * nB;
  mutual_apply_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(x, nA, nB, rowmax, colmax, out, absmax);
  P2P_LAUNCH_OK();
  return 0;
}

int launch_mutual_matching(const float* x, int nA, int nB, float* rowmax, unsigned int* colmax, float* out,
                           unsigned int* absmax, cudaStream_t st) {
  P2P_CUDA_OK(cudaMemsetAsync(colmax, 0, sizeof(unsigned int) * nB, st));
  rowcolmax_kernel<<<cdiv(nA, 8), 256, 0, st>>>(x, nA, nB, rowmax, colmax);
  P2P_LAUNCH_OK();
  return launch_mutual_apply(x, nA, nB, rowmax, colmax, out, absmax, st);
}

// ------------------------------------------------------------------------------------------------
// K5: symmetric NC conv.  conv(x) + conv(x^T)^T with shared weights equals two independent
// two-layer nets on the SAME input, the second with tap axes (a,b)<->(d,e) swapped, so layer 1
// produces 32 channels (16 per net) and layer 2 reduces each group of 16 to one map.
// hidden layout: [A cell][32][hB][wB] fp32 (HBM round trip: 2*32*V*4 B, << the FMA time).
// ------------------------------------------------------------------------------------------------
// layer 1: grid (ceil(hB/8), nA), block (ceil(wB/2), 8); thread = 2 adjacent B cells x 32 channels.
template <int MAXT, int MINB>
__global__ void __launch_bounds__(MAXT, MINB) nc_layer1_kernel(const float* __restrict__ x, int hA, int wA, int hB, int wB,
                                                       const float* __restrict__ w1p, const float* __restrict__ b1p,
                                                       float* __restrict__ hidden) {
  extern __shared__ __align__(16) float smem[];
  const int PW = wB + 4;                 // halo row pitch (>= wB+2, covers the 2-wide thread tile)
  float* w1s = smem;                     // [81][32]
  float* xs = smem + 81 * 32;            // [9][10][PW]
  const int nthreads = blockDim.x * blockDim.y;
  const int tid = threadIdx.y * blockDim.x + threadIdx.x;
  const int a = blockIdx.y, ia = a / wA, ja = a - ia * wA;
  const int k0 = blockIdx.x * 8;
  const int nB = hB * wB;
  for (int i = tid; i < 81 * 32; i += nthreads) w1s[i] = w1p[i];
  for (int i = tid; i < 9 * 10 * PW; i += nthreads) {
    const int ab = i / (10 * PW);
    const int rem = i - ab * 10 * PW;
    const int kk = rem / PW, ll = rem - kk * PW;
    const int si = ia + ab / 3 - 1, sj = ja + ab % 3 - 1;
    const int sk = k0 + kk - 1, sl = ll - 1;
    float v = 0.f;
    if (si >= 0 && si < hA && sj >= 0 && sj < wA && sk >= 0 && sk < hB && sl >= 0 && sl < wB)
      v = __ldg(x + (size_t)(si * wA + sj) * nB + sk * wB + sl);
    xs[i] = v;
  }
  __syncthreads();
  const int tl = threadIdx.x, tk = threadIdx.y;
  const int l0 = 2 * tl, k = k0 + tk;
  float acc0[32], acc1[32];
#pragma unroll
  for (int c = 0; c < 32; ++c) acc0[c] = acc1[c] = b1p[c];
  for (int ab = 0; ab < 9; ++ab) {
#pragma unroll
    for (int d = 0; d < 3; ++d) {
      const float* row = xs + (ab * 10 + tk + d) * PW + l0;
      const float v0 = row[0], v1 = row[1], v2 = row[2], v3 = row[3];
#pragma unroll
      for (int e = 0; e < 3; ++e) {
        const float u0 = e == 0 ? v0 : (e == 1 ? v1 : v2);
        const float u1 = e == 0 ? v1 : (e == 1 ? v2 : v3);
        const float4* wv = reinterpret_cast<const float4*>(w1s + (ab * 9 + d * 3 + e) * 32);
#pragma unroll
        for (int c4 = 0; c4 < 8; ++c4) {
          const float4 wq = wv[c4];
          acc0[c4 * 4 + 0] = fmaf(u0, wq.x, acc0[c4 * 4 + 0]);
          acc0[c4 * 4 + 1] = fmaf(u0, wq.y, acc0[c4 * 4 + 1]);
          acc0[c4 * 4 + 2] = fmaf(u0, wq.z, acc0[c4 * 4 + 2]);
          acc0[c4 * 4 + 3] = fmaf(u0, wq.w, acc0[c4 * 4 + 3]);
          acc1[c4 * 4 + 0] = fmaf(u1, wq.x, acc1[c4 * 4 + 0]);
          acc1[c4 * 4 + 1] = fmaf(u1, wq.y, acc1[c4 * 4 + 1]);
          acc1[c4 * 4 + 2] = fmaf(u1, wq.z, acc1[c4 * 4 + 2]);
          acc1[c4 * 4 + 3] = fmaf(u1, wq.w, acc1[c4 * 4 + 3]);
        }
      }
    }
  }
  if (k < hB) {
    float* hp = hidden + (size_t)a * 32 * nB + k * wB;
#pragma unroll
    for (int c = 0; c < 32; ++c) {
      if (l0 < wB) hp[(size_t)c * nB + l0] = fmaxf(acc0[c], 0.f);
      if (l0 + 1 < wB) hp[(size_t)c * nB + l0 + 1] = fmaxf(acc1[c], 0.f);
    }
  }
}

// layer 2: grid (nA), block (ceil(wB/4), ceil(hB/2)); thread = 2x4 B cells.  The work list is
// (net, valid A-neighbour, 4-channel group); each item stages 4 hidden planes (zero halo kept from
// initialisation) through a double-buffered cp.async pipeline and costs 288 FMAs per thread.
__device__ __forceinline__ void cp_async4(float* dst_smem, const float* src) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"((unsigned)__cvta_generic_to_shared(dst_smem)), "l"(src)
               : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

constexpr int kNc2MaxCopies = 12;   // per-thread copy slots per plane (4-byte path: ceil(hB*wB/threads) <= 8)
constexpr int kNc2Left = 4;         // interior starts at column 4 so that 16-byte cp.async rows stay aligned

__device__ __forceinline__ void cp_async16(float* dst_smem, const float* src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"((unsigned)__cvta_generic_to_shared(dst_smem)), "l"(src)
               : "memory");
}

// Row pitch of the staged planes: a multiple of 4 floats with 2*pitch = 8 (mod 32), so that the
// float4 reads of consecutive thread rows (2 plane rows apart) fall into disjoint banks.
__host__ __device__ inline int nc2_pitch(int wB) {
  int pw = kNc2Left + ((wB + 3) / 4) * 4 + 4;
  while ((2 * pw) % 32 != 8) pw += 4;
  return pw;
}

// VEC: wB % 4 == 0 -> planes are staged with 16-byte copies (4x fewer copy instructions).
// One block owns JB (<= 4) consecutive A cells of one A row: the 3 x (JB+2) neighbouring A cells'
// hidden planes are staged once and every staged plane feeds up to 3 of the JB outputs from the
// same registers (about 2x the FMAs per shared-memory load of a one-cell block).
template <bool VEC>
__global__ void __launch_bounds__(384) nc_layer2_kernel(const float* __restrict__ hidden, int hA, int wA, int hB,
                                                       int wB, int JB, const float* __restrict__ w2p, float b2,
                                                       float* __restrict__ out) {
  extern __shared__ __align__(16) float smem[];
  const int PW = nc2_pitch(wB);                       // [3 unused | left halo | interior | right halo ...]
  const int PH = hB + 2 + 1;                          // covers 2*tk+3
  const int plane = PH * PW;
  float* w2s = smem;                                  // [81][32]
  float* tile = smem + 81 * 32;                       // [2 buffers][4 planes][PH][PW]
  __shared__ int s_nb[18];
  __shared__ int s_nnb;
  const int nthreads = blockDim.x * blockDim.y;
  const int tid = threadIdx.y * blockDim.x + threadIdx.x;
  const int nJ = (wA + JB - 1) / JB;
  const int ia = blockIdx.x / nJ, j0 = (blockIdx.x - ia * nJ) * JB;
  const int nB = hB * wB;
  for (int i = tid; i < 81 * 32; i += nthreads) w2s[i] = w2p[i];
  for (int i = tid; i < 8 * plane + 16; i += nthreads) tile[i] = 0.f;   // halo stays zero for the whole kernel
  if (tid == 0) {
    int n = 0;
    for (int di = 0; di < 3; ++di)
      for (int dj = 0; dj < JB + 2; ++dj) {
        const int si = ia + di - 1, sj = j0 + dj - 1;
        if (si >= 0 && si < hA && sj >= 0 && sj < wA) s_nb[n++] = di * 6 + dj;
      }
    s_nnb = n;
  }
  // per-thread copy slots (units: 4 floats if VEC else 1 float).  Slots past the end of the plane
  // re-copy the last unit into a scratch area behind the tiles, so the copy loop needs no predicates.
  const int unit = VEC ? 4 : 1;
  const int nunits = nB / unit;
  const int wunits = wB / unit;
  const int nslots = (nunits + nthreads - 1) / nthreads;   // checked on the host
  constexpr int MAXS = VEC ? 3 : kNc2MaxCopies;
  int src_off[MAXS], dst_off[MAXS];
#pragma unroll
  for (int j = 0; j < MAXS; ++j) {
    const int e = tid + j * nthreads;
    const int ec = e < nunits ? e : nunits - 1;
    const int k = ec / wunits, l = (ec - k * wunits) * unit;
    src_off[j] = ec * unit;
    dst_off[j] = e < nunits ? (k + 1) * PW + kNc2Left + l : -1;
  }
  float* scratch = tile + 8 * plane;   // 16 floats
  __syncthreads();
  const int nnb = s_nnb;
  const int per_net = nnb * 4;
  const int nitems = 2 * per_net;
  auto issue = [&](int item) {
    const int net = item / per_net;
    const int rem = item - net * per_net;
    const int nb = s_nb[rem >> 2], cg = rem & 3;
    const int si = ia + nb / 6 - 1, sj = j0 + nb % 6 - 1;
    const float* src = hidden + ((size_t)(si * wA + sj) * 32 + net * 16 + cg * 4) * nB;
    float* dst = tile + (item & 1) * 4 * plane;
#pragma unroll
    for (int j = 0; j < MAXS; ++j) {
      if (j < nslots) {
#pragma unroll
        for (int cc = 0; cc < 4; ++cc) {
          float* d = dst_off[j] >= 0 ? dst + cc * plane + dst_off[j] : scratch;
          if (VEC)
            cp_async16(d, src + (size_t)cc * nB + src_off[j]);
          else
            cp_async4(d, src + (size_t)cc * nB + src_off[j]);
        }
      }
    }
    cp_async_commit();
  };
  const int tl = threadIdx.x, tk = threadIdx.y;
  float total[4][8], acc[4][8];
#pragma unroll
  for (int jj = 0; jj < 4; ++jj)
#pragma unroll
    for (int i = 0; i < 8; ++i) { total[jj][i] = 0.f; acc[jj][i] = b2; }
  issue(0);
  for (int item = 0; item < nitems; ++item) {
    if (item + 1 < nitems) {
      issue(item + 1);
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();
    const int net = item / per_net;
    const int rem = item - net * per_net;
    const int nb = s_nb[rem >> 2], c0 = net * 16 + (rem & 3) * 4;
    const int di = nb / 6, dj = nb - di * 6;
    const float* buf = tile + (item & 1) * 4 * plane;
#pragma unroll
    for (int cc = 0; cc < 4; ++cc) {
      float r[4][6];
#pragma unroll
      for (int rr = 0; rr < 4; ++rr) {
        const float* p = buf + cc * plane + (2 * tk + rr) * PW + 4 * tl + kNc2Left - 1;   // B column 4*tl-1
        const float4 q = *reinterpret_cast<const float4*>(p + 1);
        r[rr][0] = p[0]; r[rr][1] = q.x; r[rr][2] = q.y; r[rr][3] = q.z; r[rr][4] = q.w; r[rr][5] = p[5];
      }
#pragma unroll
      for (int jj = 0; jj < 4; ++jj) {
        const int b = dj - jj;                       // A-column tap of output jj for this neighbour
        if (jj < JB && b >= 0 && b <= 2) {           // block-uniform
          const float* wrow = w2s + (di * 3 + b) * 9 * 32 + c0 + cc;
#pragma unroll
          for (int d = 0; d < 3; ++d)
#pragma unroll
            for (int e = 0; e < 3; ++e) {
              const float wv = wrow[(d * 3 + e) * 32];
#pragma unroll
              for (int kk = 0; kk < 2; ++kk)
#pragma unroll
                for (int ll = 0; ll < 4; ++ll)
                  acc[jj][kk * 4 + ll] = fmaf(r[kk + d][ll + e], wv, acc[jj][kk * 4 + ll]);
            }
        }
      }
    }
    if (rem == per_net - 1) {   // last item of this net: ReLU and fold into the total
#pragma unroll
      for (int jj = 0; jj < 4; ++jj)
#pragma unroll
        for (int i = 0; i < 8; ++i) { total[jj][i] += fmaxf(acc[jj][i], 0.f); acc[jj][i] = b2; }
    }
    __syncthreads();             // everyone is done with this buffer before it is refilled
  }
#pragma unroll
  for (int jj = 0; jj < 4; ++jj) {
    if (jj >= JB || j0 + jj >= wA) continue;
    const size_t a = (size_t)ia * wA + j0 + jj;
#pragma unroll
    for (int kk = 0; kk < 2; ++kk)
#pragma unroll
      for (int ll = 0; ll < 4; ++ll) {
        const int k = 2 * tk + kk, l = 4 * tl + ll;
        if (k < hB && l < wB) out[a * nB + k * wB + l] = total[jj][kk * 4 + ll];
      }
  }
}

int launch_neigh_consensus(const float* x, int hA, int wA, int hB, int wB, const float* w1p, const float* b1p,
                           const float* w2p, float b2, float* hidden, float* out, cudaStream_t st) {
  const int nA = hA * wA;
  {
    dim3 block(cdiv(wB, 2), 8);
    P2P_REQUIRE(block.x * block.y <= 512, "NC layer 1: pooled width too large (wB <= 128)");
    dim3 grid(cdiv(hB, 8), nA);
    const size_t smem = sizeof(float) * (81 * 32 + 9 * 10 * (wB + 4));
    if (block.x * block.y <= 160) {   // small B grids: cap registers so that 4 blocks share an SM
      auto k = nc_layer1_kernel<160, 4>;
      P2P_ENSURE_SMEM(k, smem);
      P2P_CUDA_OK(cudaFuncSetAttribute(k, cudaFuncAttributePreferredSharedMemoryCarveout, 100));
      k<<<grid, block, smem, st>>>(x, hA, wA, hB, wB, w1p, b1p, hidden);
    } else {
      auto k = nc_layer1_kernel<512, 1>;
      P2P_ENSURE_SMEM(k, smem);
      P2P_CUDA_OK(cudaFuncSetAttribute(k, cudaFuncAttributePreferredSharedMemoryCarveout, 100));
      k<<<grid, block, smem, st>>>(x, hA, wA, hB, wB, w1p, b1p, hidden);
    }
    P2P_LAUNCH_OK();
  }
  {
    dim3 block(cdiv(wB, 4), cdiv(hB, 2));
    P2P_REQUIRE(block.x * block.y <= 384, "NC layer 2: pooled B grid too large (hB*wB <= 3072)");
    P2P_REQUIRE(cdiv(hB * wB, (int)(block.x * block.y)) <= kNc2MaxCopies, "NC layer 2: copy slots exhausted");
    P2P_REQUIRE(wB % 4 != 0 || cdiv(hB * wB / 4, (int)(block.x * block.y)) <= 3, "NC layer 2: vector copy slots exhausted");
    const int PW = nc2_pitch(wB), PH = hB + 3;
    const size_t smem = sizeof(float) * (81 * 32 + 8 * PH * PW + 16);
    P2P_REQUIRE(smem <= 200 * 1024, "NC layer 2: pooled B grid does not fit shared memory");
    // A cells per block: the choice with the least wave-quantisation waste on this device
    int JB = 2, nsm = 132;
    {
      int dev = 0;
      cudaGetDevice(&dev);
      cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, dev);
      double best = 1e30;
      for (int jb = 2; jb <= 4; ++jb) {
        const int blocks = hA * cdiv(wA, jb);
        const double per_sm = (double)blocks / nsm;
        const double waste = (double)cdiv(blocks, nsm) / per_sm * (1.0 + 0.35 / jb);   // small bonus for reuse
        if (waste < best) { best = waste; JB = jb; }
      }
    }
    const int grid = hA * cdiv(wA, JB);
    if (wB % 4 == 0) {
      P2P_ENSURE_SMEM(nc_layer2_kernel<true>, smem);
      P2P_CUDA_OK(cudaFuncSetAttribute(nc_layer2_kernel<true>, cudaFuncAttributePreferredSharedMemoryCarveout, 100));
      nc_layer2_kernel<true><<<grid, block, smem, st>>>(hidden, hA, wA, hB, wB, JB, w2p, b2, out);
    } else {
      P2P_ENSURE_SMEM(nc_layer2_kernel<false>, smem);
      P2P_CUDA_OK(cudaFuncSetAttribute(nc_layer2_kernel<false>, cudaFuncAttributePreferredSharedMemoryCarveout, 100));
      nc_layer2_kernel<false><<<grid, block, smem, st>>>(hidden, hA, wA, hB, wB, JB, w2p, b2, out);
    }
    P2P_LAUNCH_OK();
  }
  return 0;
}

// ------------------------------------------------------------------------------------------------
// K6+K7: proposals.  score = max softmax prob = 1 / sum exp(x - max); argmax with lowest-index
// ties; relocalise with the pooling code; scale to pixels.  Rows [0,nB): best A for every B cell
// (softmax over A); rows [nB, nB+nA): best B for every A cell.  Row = (x1,y1,x2,y2) int64.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ void better(float& v, int& i, float v2, int i2) {
  if (v2 > v || (v2 == v && i2 < i)) {
    v = v2;
    i = i2;
  }
}

__device__ __forceinline__ void emit_match(long long* m, float* sc, int row, int a, int b, float score, int wA, int wB,
                                           int nB, const uint8_t* code, int ks, int upsample, int shift) {
  int iA = a / wA, jA = a - iA * wA, iB = b / wB, jB = b - iB * wB;
  if (code != nullptr) {
    int c = code[(size_t)a * nB + b];
    const int dl = c % ks; c /= ks;
    const int dk = c % ks; c /= ks;
    const int dj = c % ks; c /= ks;
    iA = iA * ks + c; jA = jA * ks + dj; iB = iB * ks + dk; jB = jB * ks + dl;
  }
  m[(size_t)row * 4 + 0] = (long long)jA * upsample + shift;
  m[(size_t)row * 4 + 1] = (long long)iA * upsample + shift;
  m[(size_t)row * 4 + 2] = (long long)jB * upsample + shift;
  m[(size_t)row * 4 + 3] = (long long)iB * upsample + shift;
  sc[row] = score;
}

// best A for every B cell: block = 8 columns x 128 row phases (each thread scans nA/128 rows; nB/8 blocks cover every
// SM -- with 32 columns per block only 38 blocks existed at 640x480 and the kernel took 20 us)
__global__ void __launch_bounds__(1024) proposals_dir1_kernel(const float* __restrict__ x, int nA, int nB, int wA, int wB,
                                                             const uint8_t* __restrict__ code, int ks, int upsample,
                                                             int shift, int do_softmax, long long* __restrict__ m,
                                                             float* __restrict__ sc) {
  constexpr int C = 8, R = 128;
  __shared__ float sv[R][C + 1];
  __shared__ int si[R][C + 1];
  __shared__ float sbest[C];
  __shared__ int sbi[C];
  const int tx = threadIdx.x & (C - 1), ty = threadIdx.x / C;
  const int b = blockIdx.x * C + tx;
  float best = -INFINITY;
  int bi = 0x7fffffff;
  if (b < nB)
    for (int a = ty; a < nA; a += R) better(best, bi, x[(size_t)a * nB + b], a);
  sv[ty][tx] = best;
  si[ty][tx] = bi;
  __syncthreads();
  if (ty < 4) {                      // 4 x 8 threads: each reduces 32 phases, then thread row 0 the 4 partials
    best = sv[ty * 32][tx];
    bi = si[ty * 32][tx];
#pragma unroll 8
    for (int r = 1; r < 32; ++r) better(best, bi, sv[ty * 32 + r][tx], si[ty * 32 + r][tx]);
  }
  __syncthreads();
  if (ty < 4) {
    sv[ty][tx] = best;
    si[ty][tx] = bi;
  }
  __syncthreads();
  if (ty == 0) {
#pragma unroll
    for (int r = 1; r < 4; ++r) better(best, bi, sv[r][tx], si[r][tx]);
    sbest[tx] = best;
    sbi[tx] = bi;
  }
  __syncthreads();
  best = sbest[tx];
  bi = sbi[tx];
  float s = 0.f;
  if (b < nB && do_softmax)
    for (int a = ty; a < nA; a += R) s += expf(x[(size_t)a * nB + b] - best);
  __syncthreads();
  sv[ty][tx] = s;
  __syncthreads();
  if (ty == 0 && b < nB) {
    float tot = 0.f;
    for (int r = 0; r < R; ++r) tot += sv[r][tx];
    const float score = do_softmax ? __fdiv_rn(1.f, tot) : best;
    emit_match(m, sc, b, bi, b, score, wA, wB, nB, code, ks, upsample, shift);
  }
}

// best B for every A cell: one warp per row
__global__ void __launch_bounds__(256) proposals_dir2_kernel(const float* __restrict__ x, int nA, int nB, int wA, int wB,
                                                            const uint8_t* __restrict__ code, int ks, int upsample,
                                                            int shift, int do_softmax, long long* __restrict__ m,
                                                            float* __restrict__ sc) {
  const int lane = threadIdx.x & 31;
  const int a = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (a >= nA) return;
  const float* row = x + (size_t)a * nB;
  float best = -INFINITY;
  int bi = 0x7fffffff;
  for (int b = lane; b < nB; b += 32) better(best, bi, row[b], b);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float v2 = __shfl_xor_sync(0xffffffffu, best, o);
    const int i2 = __shfl_xor_sync(0xffffffffu, bi, o);
    better(best, bi, v2, i2);
  }
  float s = 0.f;
  if (do_softmax)
    for (int b = lane; b < nB; b += 32) s += expf(row[b] - best);
  s = warp_sum(s);
  if (lane == 0) {
    const float score = do_softmax ? __fdiv_rn(1.f, s) : best;
    emit_match(m, sc, nB + a, a, bi, score, wA, wB, nB, code, ks, upsample, shift);
  }
}

int launch_proposals(const float* corr, const uint8_t* code, int hA, int wA, int hB, int wB, int ksize, int upsample,
                     int center, int do_softmax, long long* matches, float* scores, cudaStream_t st) {
  const int nA = hA * wA, nB = hB * wB;
  const int shift = center ? upsample / 2 : 0;
  proposals_dir1_kernel<<<cdiv(nB, 8), 1024, 0, st>>>(corr, nA, nB, wA, wB, code, ksize, upsample, shift, do_softmax,
                                                      matches, scores);
  P2P_LAUNCH_OK();
  proposals_dir2_kernel<<<cdiv(nA, 8), 256, 0, st>>>(corr, nA, nB, wA, wB, code, ksize, upsample, shift, do_softmax,
                                                     matches, scores);
  P2P_LAUNCH_OK();
  return 0;
}

// ------------------------------------------------------------------------------------------------
// K8: the np.unique(axis=0, return_index, return_counts) part of filter_coarse, on the device.
// Rows are packed to 64-bit keys (4 x 16-bit coords), (key, first index) pairs are sorted by a
// single-block bitonic network, runs are detected and (for mutual) only runs of length > 1 keep
// their first-occurrence index.  Output order is lexicographic, like np.unique.
// count_out[0] = number of ids written, count_out[1] = 1 if a coordinate was out of [0,65535].
// ------------------------------------------------------------------------------------------------
// `gscratch` != nullptr: keys / indices live in global scratch instead of shared memory (candidate lists beyond
// 16384 rows, e.g. ksize 1 at 1024x768; slower, same result).
// GLOBAL = false keeps the address space of keys / idx known at compile time (ld.shared / st.shared; with a pointer that
// may be either space every access of the sort went through the generic path and the kernel was bound by it).
template <bool GLOBAL>
__global__ void __launch_bounds__(1024) unique_rows_kernel(const long long* __restrict__ rows, int n, int P, int mutual,
                                                          const float* __restrict__ scores, float thres,
                                                          int* __restrict__ ids_out, int* __restrict__ count_out,
                                                          unsigned char* gscratch) {
  extern __shared__ __align__(16) unsigned char smraw_[];
  unsigned long long* keys = GLOBAL ? reinterpret_cast<unsigned long long*>(gscratch) : reinterpret_cast<unsigned long long*>(smraw_);
  int* idx = GLOBAL ? reinterpret_cast<int*>(gscratch + (size_t)P * 8) : reinterpret_cast<int*>(smraw_ + (size_t)P * 8);
  __shared__ int s_bad;
  __shared__ int s_warp[32];
  __shared__ int s_base;
  __shared__ int s_pass_sel, s_pass_all;
  const int tid = threadIdx.x, T = blockDim.x;
  if (tid == 0) { s_bad = 0; s_base = 0; s_pass_sel = 0; s_pass_all = 0; }
  __syncthreads();
  for (int i = tid; i < P; i += T) {
    unsigned long long k = ~0ull;
    if (i < n) {
      k = 0;
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        const long long v = rows[(size_t)i * 4 + c];
        if (v < 0 || v > 65535) s_bad = 1;
        k = (k << 16) | (unsigned long long)(v & 0xffff);
      }
    }
    keys[i] = k;
    idx[i] = i;
  }
  __syncthreads();
  for (int size = 2; size <= P; size <<= 1) {
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      for (int t = tid; t < (P >> 1); t += T) {
        const int lo = ((t & ~(stride - 1)) << 1) + (t & (stride - 1));   // stride is a power of two
        const int hi = lo + stride;
        const bool asc = ((lo & size) == 0);
        const unsigned long long k0 = keys[lo], k1 = keys[hi];
        const int i0 = idx[lo], i1 = idx[hi];
        const bool gt = (k0 > k1) || (k0 == k1 && i0 > i1);
        if (gt == asc) {
          keys[lo] = k1; keys[hi] = k0;
          idx[lo] = i1; idx[hi] = i0;
        }
      }
      // pairs t in [32c, 32c + 32) touch only elements [64c, 64c + 64) while stride <= 32, and a warp always owns the
      // same pair groups: those sub-steps need warp-level ordering only (33 block barriers instead of 78 at P = 4096)
      if (stride > 32 || stride == 1) __syncthreads();
      else __syncwarp();
    }
  }
  // compaction in sorted order: chunks of T elements, block-wide exclusive scan per chunk
  for (int c0 = 0; c0 < P; c0 += T) {
    const int p = c0 + tid;
    int sel = 0;
    if (p < n) {
      const bool first = (p == 0) || (keys[p] != keys[p - 1]);
      const bool dup = (p + 1 < n) && (keys[p + 1] == keys[p]);
      sel = first && (mutual ? dup : true);
    }
    const unsigned int ball = __ballot_sync(0xffffffffu, sel);
    const int lane = tid & 31, wid = tid >> 5;
    const int wpre = __popc(ball & ((1u << lane) - 1u));
    if (lane == 0) s_warp[wid] = __popc(ball);
    __syncthreads();
    int woff = 0, tot = 0;
    for (int wv = 0; wv < (T >> 5); ++wv) {
      const int cnt = s_warp[wv];
      if (wv < wid) woff += cnt;
      tot += cnt;
    }
    const int base = s_base;
    if (sel) {
      ids_out[base + woff + wpre] = idx[p];
      if (scores != nullptr && scores[idx[p]] > thres) atomicAdd(&s_pass_sel, 1);
    }
    __syncthreads();
    if (tid == 0) s_base = base + tot;
    __syncthreads();
  }
  if (scores != nullptr) {
    int c = 0;
    for (int i = tid; i < n; i += T) c += scores[i] > thres;
    if (c) atomicAdd(&s_pass_all, c);
  }
  __syncthreads();
  if (tid == 0) {
    count_out[0] = s_base;
    count_out[1] = s_bad;
    count_out[2] = s_pass_sel;   // selected rows whose score exceeds thres
    count_out[3] = s_pass_all;   // all rows whose score exceeds thres
  }
}

// ------------------------------------------------------------------------------------------------
// K8, lists of up to kRankMaxN rows (the proposal lists of every BASELINE size): rank sort over the whole GPU instead
// of a bitonic network on one SM (62 us for 2400 rows, the other 147 SMs idle, on the critical path of the one host
// sync).  Block (bi, bj) counts, for its 256 rows i, the rows j of chunk bj that sort before them -- by (key, index)
// -- and the equal keys before / overall; the partial counts are added into zeroed scratch with atomics.  The last
// block to finish (grid-wide ticket) turns ranks into the sorted order, detects first occurrences / duplicates,
// compacts in sorted order exactly like the bitonic path, and re-zeroes the scratch for the next call.
// scratch: int rank[kRankMaxN], eqb[kRankMaxN], eqt[kRankMaxN]; unsigned ticket, bad.
// ------------------------------------------------------------------------------------------------
constexpr int kRankMaxN = 8192;

size_t unique_rank_scratch_bytes() { return (size_t)(3 * kRankMaxN + 8) * sizeof(int); }

__device__ __forceinline__ unsigned long long pack_row_key(const long long* __restrict__ rows, int i, int& bad) {
  unsigned long long k = 0;
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    const long long v = rows[(size_t)i * 4 + c];
    if (v < 0 || v > 65535) bad = 1;
    k = (k << 16) | (unsigned long long)(v & 0xffff);
  }
  return k;
}

__global__ void __launch_bounds__(256) unique_rank_kernel(const long long* __restrict__ rows, int n, int jchunk, int mutual,
                                                         const float* __restrict__ scores, float thres,
                                                         int* __restrict__ ids_out, int* __restrict__ count_out,
                                                         int* __restrict__ scratch) {
  extern __shared__ __align__(16) unsigned char smraw_[];
  unsigned long long* sk = reinterpret_cast<unsigned long long*>(smraw_);
  int* rank = scratch;
  int* eqb = scratch + kRankMaxN;
  int* eqt = scratch + 2 * kRankMaxN;
  unsigned int* ticket = reinterpret_cast<unsigned int*>(scratch + 3 * kRankMaxN);
  int* badflag = scratch + 3 * kRankMaxN + 1;
  __shared__ int s_last;
  const int tid = threadIdx.x;
  const int i = blockIdx.x * 256 + tid;
  const int j0 = blockIdx.y * jchunk, j1 = min(j0 + jchunk, n);
  int bad = 0;
  for (int j = j0 + tid; j < j1; j += 256) sk[j - j0] = pack_row_key(rows, j, bad);
  unsigned long long ki = 0;
  if (i < n) ki = pack_row_key(rows, i, bad);
  if (bad && blockIdx.y == 0) atomicOr(badflag, 1);
  __syncthreads();
  if (i < n) {
    int lt = 0, eb = 0, et = 0;
    for (int j = j0; j < j1; ++j) {
      const unsigned long long kj = sk[j - j0];        // broadcast read
      const int e = kj == ki;
      const int before = e & (j < i);
      lt += (kj < ki) | before;
      eb += before;
      et += e;
    }
    if (lt) atomicAdd(rank + i, lt);
    if (eb) atomicAdd(eqb + i, eb);
    if (et) atomicAdd(eqt + i, et);
  }
  __threadfence();
  __syncthreads();
  if (tid == 0) s_last = atomicAdd(ticket, 1u) == gridDim.x * gridDim.y - 1;
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  // ---- last block: sorted order, selection, compaction ----
  int* order = reinterpret_cast<int*>(smraw_);        // [n]
  __shared__ int s_warp[8];
  __shared__ int s_base, s_pass_sel, s_pass_all;
  if (tid == 0) { s_base = 0; s_pass_sel = 0; s_pass_all = 0; }
  for (int r = tid; r < n; r += 256) order[__ldcg(rank + r)] = r;
  __syncthreads();
  for (int c0 = 0; c0 < n; c0 += 256) {
    const int p = c0 + tid;
    int sel = 0, row = 0;
    if (p < n) {
      row = order[p];
      const bool first = __ldcg(eqb + row) == 0;
      const bool dup = __ldcg(eqt + row) > 1;
      sel = first && (mutual ? dup : true);
    }
    const unsigned int ball = __ballot_sync(0xffffffffu, sel);
    const int lane = tid & 31, wid = tid >> 5;
    const int wpre = __popc(ball & ((1u << lane) - 1u));
    if (lane == 0) s_warp[wid] = __popc(ball);
    __syncthreads();
    int woff = 0, tot = 0;
#pragma unroll
    for (int wv = 0; wv < 8; ++wv) {
      const int cnt = s_warp[wv];
      if (wv < wid) woff += cnt;
      tot += cnt;
    }
    const int base = s_base;
    if (sel) {
      ids_out[base + woff + wpre] = row;
      if (scores != nullptr && scores[row] > thres) atomicAdd(&s_pass_sel, 1);
    }
    __syncthreads();
    if (tid == 0) s_base = base + tot;
    __syncthreads();
  }
  if (scores != nullptr) {
    int c = 0;
    for (int r = tid; r < n; r += 256) c += scores[r] > thres;
    if (c) atomicAdd(&s_pass_all, c);
  }
  __syncthreads();
  if (tid == 0) {
    count_out[0] = s_base;
    count_out[1] = __ldcg(badflag);
    count_out[2] = s_pass_sel;
    count_out[3] = s_pass_all;
    *ticket = 0;
    *badflag = 0;
  }
  for (int r = tid; r < n; r += 256) { rank[r] = 0; eqb[r] = 0; eqt[r] = 0; }   // zero again for the next call
}

size_t unique_rows_scratch_bytes(int n) {
  if (n <= 16384) return 0;
  size_t P = 2;
  while (P < (size_t)n) P <<= 1;
  return P * 12;
}

int launch_unique_rows(const long long* rows, int n, int mutual, const float* scores, float thres, int* ids_out,
                       int* count_out, unsigned char* gscratch, int* rank_scratch, cudaStream_t st) {
  P2P_REQUIRE(n >= 0 && n <= (1 << 22), "unique_rows: at most 4 Mi candidate rows");
  if (n == 0) {
    P2P_CUDA_OK(cudaMemsetAsync(count_out, 0, 4 * sizeof(int), st));
    return 0;
  }
  if (n <= kRankMaxN && rank_scratch != nullptr) {
    const int bx = cdiv(n, 256);
    int by = cdiv(160, bx);                                   // >= 160 blocks in all
    if (by > cdiv(n, 32)) by = cdiv(n, 32);
    const int jchunk = cdiv(n, by);
    by = cdiv(n, jchunk);
    const size_t smem = (size_t)jchunk * 8 > (size_t)n * 4 ? (size_t)jchunk * 8 : (size_t)n * 4;
    P2P_ENSURE_SMEM(unique_rank_kernel, smem);
    unique_rank_kernel<<<dim3(bx, by), 256, smem, st>>>(rows, n, jchunk, mutual, scores, thres, ids_out, count_out, rank_scratch);
    P2P_LAUNCH_OK();
    return 0;
  }
  int P = 2;
  while (P < n) P <<= 1;
  if (n > 16384) {
    P2P_REQUIRE(gscratch != nullptr, "unique_rows: scratch missing for a large candidate list");
    unique_rows_kernel<true><<<1, 1024, 0, st>>>(rows, n, P, mutual, scores, thres, ids_out, count_out, gscratch);
  } else {
    const size_t smem = (size_t)P * 12;
    P2P_ENSURE_SMEM(unique_rows_kernel<false>, smem);
    unique_rows_kernel<false><<<1, 1024, smem, st>>>(rows, n, P, mutual, scores, thres, ids_out, count_out, nullptr);
  }
  P2P_LAUNCH_OK();
  return 0;
}

// ------------------------------------------------------------------------------------------------
// K8b: the index arithmetic of filter_coarse (networks/utils.py:51-69) + shift_to_anchors
// (networks/patch2pix.py:377-402) in one launch.  out row r <- rows[ids[sel[r]]] (sel == nullptr: identity;
// ids == nullptr: identity), scores likewise; with panc == 8 every selected row is also expanded with the
// reference's 8-row anchor template (+-pshift on point 1 with point 2 fixed, then vice versa).
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) select_anchor_kernel(const long long* __restrict__ rows,
                                                           const float* __restrict__ scores, const int* __restrict__ ids,
                                                           const int* __restrict__ sel, int m, int panc, int pshift,
                                                           long long* __restrict__ matches_out,
                                                           float* __restrict__ scores_out,
                                                           long long* __restrict__ anchors_out) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= m) return;
  int i = sel != nullptr ? sel[r] : r;
  if (ids != nullptr) i = ids[i];
  long long v[4];
#pragma unroll
  for (int c = 0; c < 4; ++c) v[c] = rows[(size_t)i * 4 + c];
  if (matches_out != nullptr) {
#pragma unroll
    for (int c = 0; c < 4; ++c) matches_out[(size_t)r * 4 + c] = v[c];
  }
  if (scores_out != nullptr) scores_out[r] = scores[i];
  if (anchors_out != nullptr && panc == 8) {
    const long long p = pshift;
#pragma unroll
    for (int t = 0; t < 8; ++t) {
      const long long sx = (t & 1) ? p : -p, sy = (t & 2) ? p : -p;
      long long* o = anchors_out + ((size_t)r * 8 + t) * 4;
      if (t < 4) { o[0] = v[0] + sx; o[1] = v[1] + sy; o[2] = v[2]; o[3] = v[3]; }
      else { o[0] = v[0]; o[1] = v[1]; o[2] = v[2] + sx; o[3] = v[3] + sy; }
    }
  }
}

int launch_select_anchor(const long long* rows, const float* scores, const int* ids, const int* sel, int m, int panc,
                         int pshift, long long* matches_out, float* scores_out, long long* anchors_out, cudaStream_t st) {
  if (m == 0) return 0;
  select_anchor_kernel<<<cdiv(m, 256), 256, 0, st>>>(rows, scores, ids, sel, m, panc, pshift, matches_out, scores_out,
                                                    anchors_out);
  P2P_LAUNCH_OK();
  return 0;
}

}  // namespace p2p
