// Refine stage, everything except the tensor-core implicit GEMMs (umma_gemm.cu):
//   feature_prep   per pair: channels-last copies of the 3 feature levels + squared-norm maps
//   patch_gather   select_local_patch_feats + patch L2 normalise + fp16 hi/lo split, written in
//                  the parity-plane layout the conv1 implicit GEMM consumes through TMA
//   fc_parse       FeatRegressNet.fc (BN folded) + parse_regressor_out
//   conv_gemm_simt CUDA-core checker for the implicit GEMMs (bring-up only)
//
// Reference semantics:
//   select_local_patch_feats        networks/utils.py:4-36
//   patch normalise / reshape       networks/patch2pix.py:173-178
//   FeatRegressNet                  networks/modules.py:56-112
//   parse_regressor_out             networks/patch2pix.py:138-155
#include "kernels.h"

namespace p2p {

// ------------------------------------------------------------------------------------------------
// feature prep
// ------------------------------------------------------------------------------------------------
// One launch for both images and all four levels: segment = (image, level); level 0 (rgb, C = 3) only needs its
// squared-norm map, levels 1..3 additionally get channels-last fp32 / level-normalised fp16 copies.
// The backbone's level l is ceil-sized (each stride-2 layer rounds up); the reference only ever indexes the top-left
// (H >> l) x (W >> l) of it (select_local_patch_feats clamps to W // ds - 1), so that crop is what gets written.
struct PrepSegment {
  const float* in;     // [C][src_h][src_w] fp32, or (fmt 1) [src_h][src_w][C] fp16
  int fmt;             // 0: NCHW fp32 (reference layout); 1: channels-last fp16 (fp16 / channels_last backbone)
  float* out;          // [npx][C] (nullptr for level 0)
  __half* out16;       // [npx][C], every pixel divided by its own norm (nullptr for level 0)
  float* nsq;          // [npx]
  int C, npx, block0;  // npx = w * (H >> l); block0 = first block of this segment
  int w, src_w, src_plane;   // cropped row width, input row pitch, input channel stride (fmt 0) in pixels
};
struct PrepArgs {
  PrepSegment seg[8];
  int nseg;
};

__global__ void __launch_bounds__(256) feature_prep_kernel(const __grid_constant__ PrepArgs a) {
  extern __shared__ float tile[];  // [C][33]
  __shared__ float part[8][32];
  __shared__ float rinv[32];
  int si = 0;
#pragma unroll
  for (int i = 1; i < 8; ++i)
    if (i < a.nseg && (int)blockIdx.x >= a.seg[i].block0) si = i;
  const PrepSegment& g = a.seg[si];
  const int C = g.C, npx = g.npx;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int px0 = ((int)blockIdx.x - g.block0) * 32;
  if (g.fmt == 1) {
    // channels-last fp16 input: one warp per pixel (4 pixels per warp and block pass), lane = C/32 channels
    const __half* in16 = reinterpret_cast<const __half*>(g.in);
    const int per = C >> 5;                 // 2 (C = 64) or 4 (C = 128) halves per lane
    for (int pp = wid; pp < 32; pp += 8) {
      const int px = px0 + pp;
      if (px >= npx) break;
      const int sp = g.src_w == g.w ? px : (px / g.w) * g.src_w + px % g.w;
      float v[4] = {0.f, 0.f, 0.f, 0.f};
      if (per == 2) {
        const float2 f = __half22float2(__ldg(reinterpret_cast<const __half2*>(in16 + (size_t)sp * C) + lane));
        v[0] = f.x; v[1] = f.y;
      } else {
        const uint2 u = __ldg(reinterpret_cast<const uint2*>(in16 + (size_t)sp * C) + lane);
        const float2 f0 = __half22float2(*reinterpret_cast<const __half2*>(&u.x)), f1 = __half22float2(*reinterpret_cast<const __half2*>(&u.y));
        v[0] = f0.x; v[1] = f0.y; v[2] = f1.x; v[3] = f1.y;
      }
      float s = 0.f;
#pragma unroll
      for (int i = 0; i < 4; ++i) s = fmaf(v[i], v[i], s);
      s = warp_sum(s);
      if (lane == 0) g.nsq[px] = s;
      const float ri = rsqrtf(s + 1e-30f);
      float* o = g.out + (size_t)px * C + lane * per;
      __half* o16 = g.out16 + (size_t)px * C + lane * per;
      for (int i = 0; i < per; ++i) {
        o[i] = v[i];
        o16[i] = __float2half_rn(v[i] * ri);
      }
    }
    return;
  }
  const int px = px0 + lane;
  const int sp = g.src_w == g.w ? px : (px / g.w) * g.src_w + px % g.w;   // crop only where the level is ceil-sized
  float s = 0.f;
  for (int c = wid; c < C; c += 8) {
    const float v = px < npx ? __ldg(g.in + (size_t)c * g.src_plane + sp) : 0.f;
    tile[c * 33 + lane] = v;
    s = fmaf(v, v, s);
  }
  part[wid][lane] = s;
  __syncthreads();
  if (wid == 0 && px < npx) {
    float t = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) t += part[w][lane];
    g.nsq[px] = t;
    rinv[lane] = rsqrtf(t + 1e-30f);
  }
  if (g.out == nullptr) return;      // block-uniform
  __syncthreads();
  for (int i = threadIdx.x; i < 32 * C; i += 256) {
    const int p = i / C, c = i - p * C;
    if (px0 + p < npx) {
      const float v = tile[c * 33 + p];
      g.out[(size_t)(px0 + p) * C + c] = v;
      g.out16[(size_t)(px0 + p) * C + c] = __float2half_rn(v * rinv[p]);   // |.| <= 1: no fp16 range issues
    }
  }
}

int launch_feature_prep_pair(const float* const feats1[4], const float* const feats2[4], const int H[2], const int W[2],
                             PairFeatures out[2], int fmt, cudaStream_t st) {
  PrepArgs a;
  memset(&a, 0, sizeof(a));
  const int chans[4] = {3, 64, 64, 128};
  int blocks = 0;
  for (int s = 0; s < 2; ++s) {
    const float* const* f = s == 0 ? feats1 : feats2;
    out[s].img = f[0];
    out[s].H = H[s];
    out[s].W = W[s];
    int src_h = H[s], src_w = W[s];
    for (int l = 0; l < 4; ++l) {
      PrepSegment& g = a.seg[a.nseg++];
      if (l > 0) {                          // ResNet's stride-2 layers: ceil(h / 2)
        src_h = (src_h + 1) >> 1;
        src_w = (src_w + 1) >> 1;
      }
      g.in = f[l];
      g.fmt = l > 0 ? fmt : 0;              // the image (level 0) is always NCHW fp32
      g.C = chans[l];
      g.w = W[s] >> l;
      g.src_w = src_w;
      g.src_plane = src_h * src_w;
      g.npx = (H[s] >> l) * g.w;
      g.nsq = out[s].nsq[l];
      g.out = l > 0 ? out[s].nhwc[l - 1] : nullptr;
      g.out16 = l > 0 ? out[s].nhwc16[l - 1] : nullptr;
      g.block0 = blocks;
      blocks += cdiv(g.npx, 32);
    }
  }
  feature_prep_kernel<<<blocks, 256, sizeof(float) * 128 * 33, st>>>(a);
  P2P_LAUNCH_OK();
  return 0;
}

// ------------------------------------------------------------------------------------------------
// Window map (fuse_gather = 3).  The 259-channel L2-normalised vector of a window pixel depends only on its absolute
// image position, so it is computed ONCE per image pixel: map[y + pad][x + pad][0..255] =
// kActScale * concat(l1, l2, l3)(y, x) / sqrt(sum_c f^2 + 1e-6), replicate-padded.  The conv1 implicit GEMM then reads
// every tap of every patch as one strided TMA box.  One warp per 8 pixels of a padded row; lane = one 16-byte channel
// chunk.  Arithmetic identical to the in-kernel producers of umma_conv1_fused_kernel (bit-identical A operand).
// select_local_patch_feats clamps per level (networks/utils.py:22-23): level l reads min(x >> l, (W >> l) - 1) for the
// full-resolution coordinate clamped to [0, W - 1].  The second bound only bites when 2^l does not divide W: for
// W = 9, x = 8 gives level-1 index 3, not 8 >> 1 = 4.
// ------------------------------------------------------------------------------------------------
struct WindowMapArgs {
  const float* img[2];
  const __half* nhwc16[2][3];
  const float* nsq[2][4];
  __half* wmap[2];
  __half* rgbn[2];
  int H[2], W[2];
  long long px0[3];     // first padded-pixel index of image 1; total
};

constexpr int kMapPxPerWarp = 8;     // consecutive pixels of one padded row (map_pitch is a multiple of 8)

__global__ void __launch_bounds__(256) window_map_kernel(const __grid_constant__ WindowMapArgs a) {
  const int lane = threadIdx.x & 31;
  const int q0 = (blockIdx.x * 8 + (threadIdx.x >> 5)) * kMapPxPerWarp;
  if (q0 >= (int)a.px0[2]) return;
  const int si = q0 >= (int)a.px0[1] ? 1 : 0;
  const int qb = q0 - (int)a.px0[si];
  const int W = a.W[si], H = a.H[si], Wp = map_pitch(W);
  const int yp = qb / Wp, xp0 = qb - yp * Wp;
  const int Y = min(max(yp - kMapPad, 0), H - 1);
  const int lvl = lane < 8 ? 0 : (lane < 16 ? 1 : 2);
  const int sh = lvl + 1, C = lvl == 2 ? 128 : 64;
  const int coff = (lane < 16 ? (lane & 7) : (lane - 16)) * 8;
  const int W1 = W >> 1, W2 = W >> 2, W3 = W >> 3, Wl = W >> sh;
  const float* nsq0 = a.nsq[si][0] + (size_t)Y * W;
  const float* nsq1 = a.nsq[si][1] + (size_t)min(Y >> 1, (H >> 1) - 1) * W1;
  const float* nsq2 = a.nsq[si][2] + (size_t)min(Y >> 2, (H >> 2) - 1) * W2;
  const float* nsq3 = a.nsq[si][3] + (size_t)min(Y >> 3, (H >> 3) - 1) * W3;
  const float* nsql = lvl == 0 ? nsq1 : (lvl == 1 ? nsq2 : nsq3);
  const __half* frow = a.nhwc16[si][lvl] + (size_t)min(Y >> sh, (H >> sh) - 1) * Wl * C + coff;
  // phase 1: every load of the warp's 8 pixels in flight; phase 2: scale and store
  uint4 v[kMapPxPerWarp];
  float t[kMapPxPerWarp], nl[kMapPxPerWarp], rgb[kMapPxPerWarp];
#pragma unroll
  for (int u = 0; u < kMapPxPerWarp; ++u) {
    const int X = min(max(xp0 + u - kMapPad, 0), W - 1);
    const int xl = min(X >> sh, Wl - 1);
    t[u] = ((__ldg(nsq0 + X) + __ldg(nsq1 + min(X >> 1, W1 - 1))) + __ldg(nsq2 + min(X >> 2, W2 - 1))) +
           __ldg(nsq3 + min(X >> 3, W3 - 1));
    nl[u] = __ldg(nsql + xl);
    v[u] = __ldg(reinterpret_cast<const uint4*>(frow + (size_t)xl * C));
    rgb[u] = lane < 3 ? __ldg(a.img[si] + ((size_t)lane * H + Y) * W + X) : 0.f;
  }
  __half* wrow = a.wmap[si] + (size_t)qb * 256;
  __half* rrow = a.rgbn[si] + (size_t)qb * 4;
#pragma unroll
  for (int u = 0; u < kMapPxPerWarp; ++u) {
    const float dinv = __fdiv_rn(kActScale, sqrtf(t[u] + 1e-6f));
    const float sc = dinv * sqrtf(nl[u] + 1e-30f);       // undo the per-level normalisation
    __half2* h2 = reinterpret_cast<__half2*>(&v[u]);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float2 f = __half22float2(h2[i]);
      h2[i] = __floats2half2_rn(f.x * sc, f.y * sc);
    }
    reinterpret_cast<uint4*>(wrow + (size_t)u * 256)[lane] = v[u];
    if (lane < 4) rrow[u * 4 + lane] = __float2half_rn(rgb[u] * dinv);
  }
}

int launch_window_map(const PairFeatures pf[2], cudaStream_t st) {
  WindowMapArgs a;
  memset(&a, 0, sizeof(a));
  long long tot = 0;
  for (int s = 0; s < 2; ++s) {
    a.img[s] = pf[s].img;
    for (int l = 0; l < 3; ++l) a.nhwc16[s][l] = pf[s].nhwc16[l];
    for (int l = 0; l < 4; ++l) a.nsq[s][l] = pf[s].nsq[l];
    a.wmap[s] = pf[s].wmap;
    a.rgbn[s] = pf[s].rgbn;
    a.H[s] = pf[s].H;
    a.W[s] = pf[s].W;
    a.px0[s] = tot;
    tot += (long long)(pf[s].H + 2 * kMapPad) * map_pitch(pf[s].W);
  }
  a.px0[2] = tot;
  window_map_kernel<<<(unsigned)((tot + 8 * kMapPxPerWarp - 1) / (8 * kMapPxPerWarp)), 256, 0, st>>>(a);
  P2P_LAUNCH_OK();
  return 0;
}

// ------------------------------------------------------------------------------------------------
// patch gather.  One block per patch.
// conv1 (k3, s2, p1) reads window pixel wx = 2*ox - 1 + tx.  Window pixels are stored in four
// parity planes so that every tap is a dense 8x8 box:  plane = py*2+px, px = 0 holds odd wx
// (entry ix <-> wx = 2*ix+1), px = 1 holds even wx (ix <-> wx = 2*ix).  Tap tx=0 -> (px 0, start -1,
// the -1 column is TMA zero fill = conv padding), tx=1 -> (px 1, start 0), tx=2 -> (px 0, start 0).
// Main tensor [N][4][8][8][512] fp16 (hi and lo), channel order
//   [img1: conv1 64 | layer1 64 | layer2 128 | img2: same];
// rgb tensor [N][64 out pixels][64] fp16 is a plain im2col of the 2x3 image channels
// (k = tap*6 + img*3 + ch; k >= 54 zero).
// ------------------------------------------------------------------------------------------------
struct GatherArgs {
  const float* img[2];
  const float* nhwc[2][3];
  const float* nsq[2][4];
  int H[2], W[2];
};

__device__ __forceinline__ int clamp_idx(int v, int ds, int full) {
  // ((x + dx) // ds).clamp(0, full // ds - 1) with Python floor division
  if (v < 0) return 0;
  const int q = v / ds, m = full / ds - 1;
  return q < m ? q : m;
}

__device__ __forceinline__ void split_store8(const float* v, __half* hi, __half* lo) {
  __align__(16) __half h[8];
  __align__(16) __half l[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    h[i] = __float2half_rn(v[i]);
    l[i] = __float2half_rn(v[i] - __half2float(h[i]));
  }
  *reinterpret_cast<uint4*>(hi) = *reinterpret_cast<const uint4*>(h);
  if (lo != nullptr) *reinterpret_cast<uint4*>(lo) = *reinterpret_cast<const uint4*>(l);
}

template <bool IS_FLOAT>
__global__ void __launch_bounds__(256) patch_gather_kernel(GatherArgs g, const void* __restrict__ matches, int N,
                                                          __half* __restrict__ p_hi, __half* __restrict__ p_lo,
                                                          __half* __restrict__ rgb_hi, __half* __restrict__ rgb_lo,
                                                          const int* __restrict__ rowmap,
                                                          const int* __restrict__ d_count) {
  __shared__ float dinv[2][16][16];  // act_scale / sqrt(sum_c f^2 + 1e-6) per window pixel
  __shared__ int org[4];
  const int n = blockIdx.x;          // patch slot
  if (d_count != nullptr && n >= *d_count) return;
  const int row = rowmap != nullptr ? rowmap[n] : n;
  const int tid = threadIdx.x;
  if (tid < 4) {
    int v;
    if (IS_FLOAT)
      v = (int)reinterpret_cast<const float*>(matches)[(size_t)row * 4 + tid];  // .long(): truncation
    else
      v = (int)reinterpret_cast<const long long*>(matches)[(size_t)row * 4 + tid];
    org[tid] = v - 8;
  }
  __syncthreads();
  for (int i = tid; i < 512; i += 256) {
    const int s = i >> 8, wy = (i >> 4) & 15, wx = i & 15;
    const int X = org[2 * s] + wx, Y = org[2 * s + 1] + wy;
    float t = 0.f;
#pragma unroll
    for (int l = 0; l < 4; ++l) {
      const int ds = 1 << l;
      const int xi = clamp_idx(X, ds, g.W[s]), yi = clamp_idx(Y, ds, g.H[s]);
      t += __ldg(g.nsq[s][l] + (size_t)yi * (g.W[s] / ds) + xi);
    }
    dinv[s][wy][wx] = __fdiv_rn(kActScale, sqrtf(t + 1e-6f));
  }
  __syncthreads();
  // main channels: one warp per window position.  Lane l owns channels [8l, 8l+8) of image 1 AND
  // of image 2, so every warp store instruction covers one contiguous 512-byte row segment.
  const int lane = tid & 31, wid = tid >> 5;
  const int jj = lane >> 3;                          // 64-channel chunk inside one image's 256
  const int lvl = jj == 0 ? 0 : (jj == 1 ? 1 : 2);   // index into nhwc[] (feature levels 1..3)
  const int ds = 2 << lvl;
  const int C = lvl == 2 ? 128 : 64;
  const int coff = (jj == 3 ? 64 : 0) + (lane & 7) * 8;
  for (int pos0 = wid; pos0 < kPatchPos; pos0 += 16) {
    float4 t[2][2][2];
    float sc[2][2];
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      const int pos = pos0 + 8 * u;
      const int plane = pos >> 6, iy = (pos >> 3) & 7, ix = pos & 7;
      const int wx = (plane & 1) ? 2 * ix : 2 * ix + 1;
      const int wy = (plane & 2) ? 2 * iy : 2 * iy + 1;
#pragma unroll
      for (int s = 0; s < 2; ++s) {
        const int xi = clamp_idx(org[2 * s] + wx, ds, g.W[s]), yi = clamp_idx(org[2 * s + 1] + wy, ds, g.H[s]);
        sc[u][s] = dinv[s][wy][wx];
        const float4* src =
            reinterpret_cast<const float4*>(g.nhwc[s][lvl] + ((size_t)yi * (g.W[s] / ds) + xi) * C + coff);
        t[u][s][0] = __ldg(src);
        t[u][s][1] = __ldg(src + 1);
      }
    }
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      const int pos = pos0 + 8 * u;
#pragma unroll
      for (int s = 0; s < 2; ++s) {
        const float k = sc[u][s];
        const float v[8] = {t[u][s][0].x * k, t[u][s][0].y * k, t[u][s][0].z * k, t[u][s][0].w * k,
                            t[u][s][1].x * k, t[u][s][1].y * k, t[u][s][1].z * k, t[u][s][1].w * k};
        const size_t o = ((size_t)n * kPatchPos + pos) * kMainCh + s * 256 + lane * 8;
        split_store8(v, p_hi + o, p_lo ? p_lo + o : nullptr);
      }
    }
  }
  // rgb im2col: 64 output pixels x 64 k
  for (int e = tid; e < 64 * 64; e += 256) {
    const int o = e >> 6, k = e & 63;
    float v = 0.f;
    if (k < 54) {
      const int tap = k / 6, r = k - tap * 6;
      const int si = r / 3, ch = r - si * 3;
      const int wx = 2 * (o & 7) - 1 + tap % 3, wy = 2 * (o >> 3) - 1 + tap / 3;
      if (wx >= 0 && wy >= 0) {
        const int xi = clamp_idx(org[2 * si] + wx, 1, g.W[si]), yi = clamp_idx(org[2 * si + 1] + wy, 1, g.H[si]);
        v = __ldg(g.img[si] + ((size_t)ch * g.H[si] + yi) * g.W[si] + xi) * dinv[si][wy][wx];
      }
    }
    const __half h = __float2half_rn(v);
    const size_t oi = (size_t)n * 4096 + e;
    rgb_hi[oi] = h;
    if (rgb_lo) rgb_lo[oi] = __float2half_rn(v - __half2float(h));
  }
}

int launch_patch_gather(const PairFeatures& f1, const PairFeatures& f2, const void* matches, int is_float, int N,
                        __half* p_hi, __half* p_lo, __half* rgb_hi, __half* rgb_lo, const int* rowmap,
                        const int* d_count, cudaStream_t st) {
  if (N == 0) return 0;
  GatherArgs g;
  const PairFeatures* f[2] = {&f1, &f2};
  for (int s = 0; s < 2; ++s) {
    g.img[s] = f[s]->img;
    for (int l = 0; l < 3; ++l) g.nhwc[s][l] = f[s]->nhwc[l];
    for (int l = 0; l < 4; ++l) g.nsq[s][l] = f[s]->nsq[l];
    g.H[s] = f[s]->H;
    g.W[s] = f[s]->W;
  }
  if (is_float)
    patch_gather_kernel<true><<<N, 256, 0, st>>>(g, matches, N, p_hi, p_lo, rgb_hi, rgb_lo, rowmap, d_count);
  else
    patch_gather_kernel<false><<<N, 256, 0, st>>>(g, matches, N, p_hi, p_lo, rgb_hi, rgb_lo, rowmap, d_count);
  P2P_LAUNCH_OK();
  return 0;
}

// ------------------------------------------------------------------------------------------------
// FC stack + parse_regressor_out.  8 patches per block; weights transposed [in][out] so that the
// per-k weight reads of a warp are coalesced; 5 blocks per SM hide the L2 latency of those reads.
// (A shared-memory staged cp.async variant and a 16-patch variant were measured slower: 0.16-0.18 ms
// vs 0.11 ms per 3200 patches.)
// ------------------------------------------------------------------------------------------------
template <bool IS_FLOAT>
__global__ void __launch_bounds__(256) fc_parse_kernel(const float* __restrict__ pooled, FcWeights fc,
                                                      const void* __restrict__ matches_in, int N, float W1, float H1,
                                                      float W2, float H2, float* __restrict__ matches_out,
                                                      float* __restrict__ probs_out, float* __restrict__ raw_out,
                                                      const int* __restrict__ rowmap, const int* __restrict__ d_count) {
  constexpr int PB = 8;
  if (d_count != nullptr) {
    N = *d_count;
    if ((int)blockIdx.x * PB >= N) return;
  }
  __shared__ __align__(16) float xs[512][PB];
  __shared__ __align__(16) float h1[512][PB];
  __shared__ __align__(16) float h2[256][PB];
  __shared__ float o5[5][PB];
  const int t = threadIdx.x;
  const int n0 = blockIdx.x * PB;
  for (int i = t; i < 512 * PB; i += 256) {
    const int p = i / 512, k = i - p * 512;
    xs[k][p] = (n0 + p < N) ? pooled[(size_t)(n0 + p) * 512 + k] : 0.f;
  }
  __syncthreads();
  {
    float a0[PB], a1[PB];
#pragma unroll
    for (int p = 0; p < PB; ++p) { a0[p] = 0.f; a1[p] = 0.f; }
#pragma unroll 8
    for (int k = 0; k < 512; ++k) {
      const float w0 = __ldg(fc.w1t + (size_t)k * 512 + t), w1 = __ldg(fc.w1t + (size_t)k * 512 + t + 256);
      const float4 xa = *reinterpret_cast<const float4*>(&xs[k][0]);
      const float4 xb = *reinterpret_cast<const float4*>(&xs[k][4]);
      const float xv[PB] = {xa.x, xa.y, xa.z, xa.w, xb.x, xb.y, xb.z, xb.w};
#pragma unroll
      for (int p = 0; p < PB; ++p) { a0[p] = fmaf(xv[p], w0, a0[p]); a1[p] = fmaf(xv[p], w1, a1[p]); }
    }
    const float b0 = fc.b1[t], b1 = fc.b1[t + 256];
#pragma unroll
    for (int p = 0; p < PB; ++p) { h1[t][p] = fmaxf(a0[p] + b0, 0.f); h1[t + 256][p] = fmaxf(a1[p] + b1, 0.f); }
  }
  __syncthreads();
  {
    float a[PB];
#pragma unroll
    for (int p = 0; p < PB; ++p) a[p] = 0.f;
#pragma unroll 8
    for (int k = 0; k < 512; ++k) {
      const float w = __ldg(fc.w2t + (size_t)k * 256 + t);
      const float4 xa = *reinterpret_cast<const float4*>(&h1[k][0]);
      const float4 xb = *reinterpret_cast<const float4*>(&h1[k][4]);
      const float xv[PB] = {xa.x, xa.y, xa.z, xa.w, xb.x, xb.y, xb.z, xb.w};
#pragma unroll
      for (int p = 0; p < PB; ++p) a[p] = fmaf(xv[p], w, a[p]);
    }
    const float b = fc.b2[t];
#pragma unroll
    for (int p = 0; p < PB; ++p) h2[t][p] = fmaxf(a[p] + b, 0.f);
  }
  __syncthreads();
  if (t < 5 * PB) {
    const int o = t / PB, p = t - o * PB;
    float a = 0.f;
    for (int k = 0; k < 256; ++k) a = fmaf(h2[k][p], __ldg(fc.w3t + k * 5 + o), a);
    o5[o][p] = a + fc.b3[o];
  }
  __syncthreads();
  if (t < 5 * PB) {
    const int j = t / PB, p = t - j * PB;
    if (n0 + p < N) {
      const int n = rowmap != nullptr ? rowmap[n0 + p] : n0 + p;   // output row
      const float o = o5[j][p];
      if (raw_out != nullptr) raw_out[(size_t)n * 5 + j] = o;
      if (j < 4) {
        float m;
        if (IS_FLOAT)
          m = reinterpret_cast<const float*>(matches_in)[(size_t)n * 4 + j];
        else
          m = (float)reinterpret_cast<const long long*>(matches_in)[(size_t)n * 4 + j];
        const float off = 16.f * tanhf(fmaxf(o, 0.f)) - 8.f;
        const float hi = (j == 0) ? W1 : (j == 1) ? H1 : (j == 2) ? W2 : H2;
        matches_out[(size_t)n * 4 + j] = fminf(fmaxf(m + off, 0.f), hi);
      } else {
        probs_out[n] = __fdiv_rn(1.f, 1.f + expf(-o));
      }
    }
  }
}

int launch_fc_parse(const float* pooled, const FcWeights& fc, const void* matches_in, int is_float, int N, int W1,
                    int H1, int W2, int H2, float* matches_out, float* probs_out, float* raw_out, const int* rowmap,
                    const int* d_count, cudaStream_t st) {
  if (N == 0) return 0;
  if (is_float)
    fc_parse_kernel<true><<<cdiv(N, 8), 256, 0, st>>>(pooled, fc, matches_in, N, (float)W1, (float)H1, (float)W2,
                                                     (float)H2, matches_out, probs_out, raw_out, rowmap, d_count);
  else
    fc_parse_kernel<false><<<cdiv(N, 8), 256, 0, st>>>(pooled, fc, matches_in, N, (float)W1, (float)H1, (float)W2,
                                                      (float)H2, matches_out, probs_out, raw_out, rowmap, d_count);
  P2P_LAUNCH_OK();
  return 0;
}

// ------------------------------------------------------------------------------------------------
// Tensor-core FC path: the two big Linear layers run on umma_gemm_kernel<EPI_FC> (3-pass, fp32-grade);
// these two kernels are its prologue (pooled -> fp16 hi/lo) and tail (Linear(256,5) + parse_regressor_out).
// ------------------------------------------------------------------------------------------------
__global__ void pooled_split_kernel(const float* __restrict__ pooled, int n, float scale, __half* __restrict__ hi,
                                    __half* __restrict__ lo, const int* __restrict__ d_count) {
  if (d_count != nullptr) n = *d_count;
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)n * 512) return;
  const float v = fminf(pooled[i] * scale, 65504.f);   // pooled >= 0 (post-ReLU); saturate, never inf/NaN
  const __half h = __float2half_rn(v);
  hi[i] = h;
  lo[i] = __float2half_rn(v - __half2float(h));
}

int launch_pooled_split(const float* pooled, int n, float scale, __half* hi, __half* lo, const int* d_count, cudaStream_t st) {
  if (n == 0) return 0;
  pooled_split_kernel<<<(unsigned)(((size_t)n * 512 + 255) / 256), 256, 0, st>>>(pooled, n, scale, hi, lo, d_count);
  P2P_LAUNCH_OK();
  return 0;
}

// one warp per row: 5 dot products of length 256, then parse_regressor_out (networks/patch2pix.py:138-155)
template <bool IS_FLOAT>
__global__ void __launch_bounds__(256) fc3_parse_kernel(const __half* __restrict__ h2_hi, const __half* __restrict__ h2_lo,
                                                       float inv_scale, const float* __restrict__ w3t, const float* __restrict__ b3,
                                                       const void* __restrict__ matches_in, int N, float W1, float H1,
                                                       float W2, float H2, float* __restrict__ matches_out,
                                                       float* __restrict__ probs_out, float* __restrict__ raw_out,
                                                       const int* __restrict__ rowmap, const int* __restrict__ d_count) {
  if (d_count != nullptr) N = *d_count;
  const int lane = threadIdx.x & 31;
  const int slot = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (slot >= N) return;
  float acc[5] = {0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int k = lane + 32 * i;
    const float x = (__half2float(h2_hi[(size_t)slot * 256 + k]) + __half2float(h2_lo[(size_t)slot * 256 + k])) * inv_scale;
#pragma unroll
    for (int o = 0; o < 5; ++o) acc[o] = fmaf(x, __ldg(w3t + k * 5 + o), acc[o]);
  }
#pragma unroll
  for (int o = 0; o < 5; ++o) acc[o] = warp_sum(acc[o]);
  if (lane < 5) {
    const int n = rowmap != nullptr ? rowmap[slot] : slot;
    const int j = lane;
    const float o = (j == 0 ? acc[0] : j == 1 ? acc[1] : j == 2 ? acc[2] : j == 3 ? acc[3] : acc[4]) + b3[j];
    if (raw_out != nullptr) raw_out[(size_t)n * 5 + j] = o;
    if (j < 4) {
      float m;
      if (IS_FLOAT)
        m = reinterpret_cast<const float*>(matches_in)[(size_t)n * 4 + j];
      else
        m = (float)reinterpret_cast<const long long*>(matches_in)[(size_t)n * 4 + j];
      const float off = 16.f * tanhf(fmaxf(o, 0.f)) - 8.f;
      const float hi = (j == 0) ? W1 : (j == 1) ? H1 : (j == 2) ? W2 : H2;
      matches_out[(size_t)n * 4 + j] = fminf(fmaxf(m + off, 0.f), hi);
    } else {
      probs_out[n] = __fdiv_rn(1.f, 1.f + expf(-o));
    }
  }
}

int launch_fc3_parse(const __half* h2_hi, const __half* h2_lo, float inv_scale, const float* w3t, const float* b3, const void* matches_in,
                     int is_float, int N, int W1, int H1, int W2, int H2, float* matches_out, float* probs_out,
                     float* raw_out, const int* rowmap, const int* d_count, cudaStream_t st) {
  if (N == 0) return 0;
  if (is_float)
    fc3_parse_kernel<true><<<cdiv(N, 8), 256, 0, st>>>(h2_hi, h2_lo, inv_scale, w3t, b3, matches_in, N, (float)W1, (float)H1,
                                                      (float)W2, (float)H2, matches_out, probs_out, raw_out, rowmap,
                                                      d_count);
  else
    fc3_parse_kernel<false><<<cdiv(N, 8), 256, 0, st>>>(h2_hi, h2_lo, inv_scale, w3t, b3, matches_in, N, (float)W1, (float)H1,
                                                       (float)W2, (float)H2, matches_out, probs_out, raw_out, rowmap,
                                                       d_count);
  P2P_LAUNCH_OK();
  return 0;
}

// ------------------------------------------------------------------------------------------------
// Risk band: the fine stage gathers around trunc(mid).  A row needs fp32-grade mid arithmetic only
// if one of its coordinates lies within tau px of an integer; coordinates whose raw output is
// clearly negative get the exact offset -8 in any precision and are never at risk.
// Single block, order-preserving compaction.
// ------------------------------------------------------------------------------------------------
template <bool IS_FLOAT>
__global__ void __launch_bounds__(1024) flag_risky_kernel(const void* __restrict__ matches_in,
                                                         const float* __restrict__ raw, int N, float tau, float eps_o,
                                                         float W1, float H1, float W2, float H2,
                                                         int* __restrict__ rowmap, int* __restrict__ d_count,
                                                         unsigned long long* __restrict__ totals) {
  __shared__ int s_warp[32];
  __shared__ int s_base;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  if (tid == 0) s_base = 0;
  __syncthreads();
  for (int r0 = 0; r0 < N; r0 += 1024) {
    const int r = r0 + tid;
    int risky = 0;
    if (r < N) {
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float o = raw[(size_t)r * 5 + j];
        if (o <= -eps_o) continue;                       // offset is exactly -8 in any precision
        float m;
        if (IS_FLOAT)
          m = reinterpret_cast<const float*>(matches_in)[(size_t)r * 4 + j];
        else
          m = (float)reinterpret_cast<const long long*>(matches_in)[(size_t)r * 4 + j];
        const float th = tanhf(fmaxf(o, 0.f));
        const float v = m + (16.f * th - 8.f);           // un-clamped coordinate
        const float hi = (j == 0) ? W1 : (j == 1) ? H1 : (j == 2) ? W2 : H2;
        if (v <= -tau || v >= hi + tau) continue;        // clamped to the same bound on both sides
        // a 1-pass error do of the raw output moves the coordinate by 16 * sech^2(o) * do: the band
        // (tau at o = 0) shrinks with the tanh slope, plus a floor for fp32 rounding of the coordinate
        const float band = fminf(tau, tau * (1.f - th * th) + 3e-4f);
        if (fabsf(v - rintf(v)) < band) risky = 1;
      }
    }
    const unsigned int ball = __ballot_sync(0xffffffffu, risky);
    if (lane == 0) s_warp[wid] = __popc(ball);
    __syncthreads();
    int woff = 0, tot = 0;
    for (int w = 0; w < 32; ++w) {
      const int c = s_warp[w];
      if (w < wid) woff += c;
      tot += c;
    }
    const int base = s_base;
    if (risky) rowmap[base + woff + __popc(ball & ((1u << lane) - 1u))] = r;
    __syncthreads();
    if (tid == 0) s_base = base + tot;
    __syncthreads();
  }
  if (tid == 0) {
    *d_count = s_base;
    if (totals != nullptr) {         // running totals over calls (bench.py: band rows / rows, without a per-step sync)
      atomicAdd(totals, (unsigned long long)s_base);
      atomicAdd(totals + 1, (unsigned long long)N);
    }
  }
}

int launch_flag_risky(const void* matches_in, int is_float, const float* raw, int N, float tau, float eps_o, int W1,
                      int H1, int W2, int H2, int* rowmap, int* d_count, unsigned long long* totals, cudaStream_t st) {
  if (is_float)
    flag_risky_kernel<true><<<1, 1024, 0, st>>>(matches_in, raw, N, tau, eps_o, (float)W1, (float)H1, (float)W2,
                                                (float)H2, rowmap, d_count, totals);
  else
    flag_risky_kernel<false><<<1, 1024, 0, st>>>(matches_in, raw, N, tau, eps_o, (float)W1, (float)H1, (float)W2,
                                                 (float)H2, rowmap, d_count, totals);
  P2P_LAUNCH_OK();
  return 0;
}

// ------------------------------------------------------------------------------------------------
// Tail of estimate_matches (utils/eval/model_helper.py:97-109) on the device: inlier filter
// `scores > io_thres` (keep everything if nothing passes), order preserved, and the rescaling to original-image
// pixels `upscale * matches` in float64 (numpy promotes float32 / int64 times a float64 array to float64).
// packed [N][9] doubles = (x1,y1,x2,y2 refined, score, x1,y1,x2,y2 coarse); packed[N*9] = number of rows kept.
// fine == nullptr (eval_type 'coarse'): the refined columns repeat the coarse ones.  Single block.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(1024) finalize_matches_kernel(const float* __restrict__ fine, const float* __restrict__ scores,
                                                               const long long* __restrict__ coarse, int N, float io_thres,
                                                               double u0, double u1, double u2, double u3,
                                                               double* __restrict__ packed) {
  __shared__ int s_warp[32];
  __shared__ int s_base, s_any;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  if (tid == 0) { s_base = 0; s_any = 0; }
  __syncthreads();
  int any = 0;
  for (int r = tid; r < N; r += 1024) any |= scores[r] > io_thres;
  if (any) s_any = 1;
  __syncthreads();
  const bool keep_all = s_any == 0;
  const double up[4] = {u0, u1, u2, u3};
  for (int r0 = 0; r0 < N; r0 += 1024) {
    const int r = r0 + tid;
    const int sel = r < N && (keep_all || scores[r] > io_thres);
    const unsigned int ball = __ballot_sync(0xffffffffu, sel);
    if (lane == 0) s_warp[wid] = __popc(ball);
    __syncthreads();
    int woff = 0, tot = 0;
    for (int w = 0; w < 32; ++w) {
      const int c = s_warp[w];
      if (w < wid) woff += c;
      tot += c;
    }
    const int base = s_base;
    if (sel) {
      double* o = packed + (size_t)(base + woff + __popc(ball & ((1u << lane) - 1u))) * 9;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const double c = (double)coarse[(size_t)r * 4 + j];
        o[5 + j] = up[j] * c;
        o[j] = fine != nullptr ? up[j] * (double)fine[(size_t)r * 4 + j] : up[j] * c;
      }
      o[4] = (double)scores[r];
    }
    __syncthreads();
    if (tid == 0) s_base = base + tot;
    __syncthreads();
  }
  if (tid == 0) packed[(size_t)N * 9] = (double)s_base;
}

int launch_finalize_matches(const float* fine, const float* scores, const long long* coarse, int N, float io_thres,
                            const double up[4], double* packed, cudaStream_t st) {
  finalize_matches_kernel<<<1, 1024, 0, st>>>(fine, scores, coarse, N, io_thres, up[0], up[1], up[2], up[3], packed);
  P2P_LAUNCH_OK();
  return 0;
}

// ------------------------------------------------------------------------------------------------
// CUDA-core checker GEMM (bring-up only).  Tile 128 rows (2 patches) x 64 output channels.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) conv_gemm_simt_kernel(GemmOperands g, ConvEpilogue e) {
  __shared__ float As[32][129];
  __shared__ float Bs[32][65];
  const int tid = threadIdx.x;
  const int n0 = blockIdx.x * 2, o0 = blockIdx.y * 64;
  const int tx = tid & 15, ty = tid >> 4;  // cols tx*4.., rows ty*8..
  float acc[8][4];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  for (int si = 0; si < g.nsteps; ++si) {
    const KStep ks = g.steps[si];
    for (int half = 0; half < 2; ++half) {
      __syncthreads();
      for (int i = tid; i < 128 * 32; i += 256) {
        const int row = i >> 5, kk = (i & 31) + half * 32;
        const int n = n0 + (row >> 6), py = (row >> 3) & 7, px = row & 7;
        float v = 0.f;
        if (n < g.n_patches) {
          if (ks.kind == 1) {
            const size_t a = ((size_t)n * 64 + (row & 63)) * 64 + kk;
            v = __half2float(g.r_hi[a]);
            if (g.passes == 3) v += __half2float(g.r_lo[a]);
          } else {
            const int x = px + ks.x, y = py + ks.y;
            if (x >= 0 && x < 8 && y >= 0 && y < 8) {
              const size_t a = ((((size_t)n * g.planes + ks.plane) * 8 + y) * 8 + x) * 512 + ks.c0 + kk;
              v = __half2float(g.a_hi[a]);
              if (g.passes == 3) v += __half2float(g.a_lo[a]);
            }
          }
        }
        As[i & 31][row] = v;
      }
      for (int i = tid; i < 64 * 32; i += 256) {
        const int col = i >> 5, kk = (i & 31) + half * 32;
        const size_t b = (size_t)(o0 + col) * g.ktot + ks.bk + kk;
        float v = __half2float(g.b_hi[b]);
        if (g.passes == 3) v += __half2float(g.b_lo[b]);
        Bs[i & 31][col] = v;
      }
      __syncthreads();
#pragma unroll 4
      for (int kk = 0; kk < 32; ++kk) {
        float a[8], b[4];
#pragma unroll
        for (int i = 0; i < 8; ++i) a[i] = As[kk][ty * 8 + i];
#pragma unroll
        for (int j = 0; j < 4; ++j) b[j] = Bs[kk][tx * 4 + j];
#pragma unroll
        for (int i = 0; i < 8; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
      }
    }
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int row = ty * 8 + i;
    const int n = n0 + (row >> 6);
    if (n >= g.n_patches) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int o = o0 + tx * 4 + j;
      const float y = fmaf(acc[i][j], e.scale[o], e.bias[o]);
      if (e.mode == 0) {
        const float v = y * e.y_scale;
        const __half h = __float2half_rn(v);
        const size_t a = ((size_t)n * 64 + (row & 63)) * 512 + o;
        e.y_hi[a] = h;
        if (e.y_lo) e.y_lo[a] = __float2half_rn(v - __half2float(h));
      } else {
        atomicMax(reinterpret_cast<unsigned int*>(e.pooled) + (size_t)n * 512 + o, __float_as_uint(fmaxf(y, 0.f)));
      }
    }
  }
}

int launch_conv_gemm_simt(const GemmOperands& g, const ConvEpilogue& e, cudaStream_t st) {
  if (g.n_patches == 0) return 0;
  if (e.mode == 1) P2P_CUDA_OK(cudaMemsetAsync(e.pooled, 0, sizeof(float) * 512 * (size_t)g.n_patches, st));
  dim3 grid(cdiv(g.n_patches, 2), 8);
  conv_gemm_simt_kernel<<<grid, 256, 0, st>>>(g, e);
  P2P_LAUNCH_OK();
  return 0;
}

}  // namespace p2p
