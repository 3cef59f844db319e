// General NeighConsensus stack (NCNet's ImMatchNet: L Conv4d layers, kernel 3 or 5 per layer, 1..16 channels, the last
// layer 1 channel, bias + ReLU after every layer, symmetric or not) on the Hopper tensor cores (wgmma).
//
// Reference semantics (file:line relative to the reference repo):
//   NeighConsensus.forward   networks/ncn/model.py:124-155   conv(x) + conv(x^T)^T in symmetric mode
//   Conv4d / conv4d          networks/ncn/conv4d.py:12-74    true 4D cross-correlation, zero "same" padding of k/2
//
// Symmetric mode runs two nets on the SAME input, net 1 with the A and B tap axes swapped in every layer:
// stack(x^T)^T is the stack of the transposed filters applied to x, because transposition commutes with the
// element-wise bias + ReLU between the layers.
//
// Every layer runs one kernel, nc_stack_layer_kernel, on a uniform cell format:
//   line      one 128-byte line per 4D cell = 64 fp16 = [net 0 hi 16 ch | net 0 lo 16 ch | net 1 hi 16 | net 1 lo 16]
//             of the layer's input scaled by a power of two; channels past the layer's input count are 0.  The first
//             layer's input (1 channel) is packed into this format by nc_stack_pack_kernel (channel 0 only).
//   tile      128 MMA rows = R rows x TW columns of one A cell's B grid, enumerated with pitch P = TW + 2p lines
//             (p = k/2); the two MMA rows per tile row that fall on the column halo are junk and skipped.
//   A-taps    for each of the k^2 A-neighbours a' of the tile's A cell that lies inside the A grid (the others
//             contribute zero), a tensor-map load brings a' 's block of lines -- rows k0-p .. k0+R+p-1, columns
//             l0-p .. l0+TW+p-1, zero-filled outside the B grid -- into shared memory, 128B-swizzled as wgmma reads it.
//   B-taps    the A operand of B-tap (tk, tl) is that block starting (tk * P + tl) lines further on (a 128-byte granular
//             descriptor start, as in nc_umma.cu layer 2), so no producer warps build operands.
//   weights   per (A-tap, B-tap): a [32 rows][64] K-major image, rows 0..15 = w_hi of output channel co, 16..31 = w_lo,
//             column net * 16 + ci (one K16 slice per net).  They stream in per (A-tap, B-tap row tk): k images per
//             ring stage, bulk-copied by the loader thread next to the blocks (a k^4 x 4 KB layer does not fit in
//             shared memory).
//   MMAs      per tap and net: a_hi x [w_hi | w_lo] (N = 32: hi*hi and hi*lo) and a_lo x w_hi (N = 16: lo*hi).
//   restart   the accumulators restart at every A-tap: one chain is k^2 MMAs of K = 16, and the per-A-tap sums are
//             added to fp32 register totals in a fixed order (the tensor core truncates on every accumulate, so a
//             625 x 16-long chain would lose bits).
//   epilogue  + bias, ReLU; hidden layers re-scale and split into the next layer's lines, the last layer writes
//             out = relu(net 0) + relu(net 1) in fp32.
//
// Scales: the activations of layer l are bounded by B_l = max_c (sum |w_l[c]| * B_(l-1) + |b_l[c]|), B_0 = max|x|
// (a weight-norm bound, as nc_scales does for the fixed stack), evaluated on the device from max|x| and per-channel
// sums packed on the host.  Each layer's input is scaled by the power of two that puts its bound in [2048, 4096), so
// no fp16 operand overflows whatever the input range; weights are scaled so that max|w| lands in [512, 1024).
//
// Persistent launch: grid = min(tiles, SMs); every tile is computed by one CTA in a fixed order, so the result does not
// depend on the grid.  384 threads: warp 3 loader, warpgroups 1 and 2 = MMA rows 0..63 and 64..127 + epilogue.
#include <math.h>

#include <vector>

#include "kernels.h"
#include "umma_gemm.h"
#include "umma_ptx.cuh"

namespace p2p {

constexpr int kStackRing = 8;           // upper bound of either ring's depth (barrier arrays)
constexpr int kStackWTap = 32 * 128;    // weight image of one (A-tap, B-tap)
constexpr int kStackSmemBudget = 220 * 1024;

struct NcStackLayerParams {
  int hA, wA, hB, wB, nA, nB;
  int k, p;                     // kernel size, k / 2
  int cout;                     // output channels of this layer
  int layer;                    // index in the stack (scale chain)
  int last;                     // 1: write fp32 out, 0: write the next layer's lines
  int TW, R, P, KB, LB, tiles;  // tiling of the B grid (see above)
  int ring_b, unit_b;           // block ring: stages, bytes per stage
  int ring_w;                   // weight ring stages (k images each)
  const __half* wimg;           // [k^2 A-taps][k tk][k tl][32][64] swizzled images
  const float* bias;            // [16]
  const float* bnd;             // [layers][2][16]: per output channel sum |w|, |b|
  float inv_sw;                 // 1 / weight scale
  const unsigned int* xmax;     // float bits of max |x|
  __half* out_lines;            // [nA * nB][64] (hidden layers)
  float* out;                   // [nA * nB] (last layer)
};

// power of two s with bound * s in [2048, 4096)
__device__ __forceinline__ float stack_scale(float bound) {
  if (!(bound > 0.f) || !isfinite(bound)) bound = 1.f;
  int e;
  frexpf(bound, &e);
  return ldexpf(1.f, min(12 - e, 60));
}

// scales of the input (s_in) and output (s_out) activations of layer `layer`
__device__ __forceinline__ void stack_scales(const float* bnd, const unsigned int* xmax, int layer, float& s_in, float& s_out) {
  float b = __uint_as_float(__ldg(xmax));
  if (!(b > 0.f) || !isfinite(b)) b = 1.f;
  s_in = stack_scale(b);
  for (int l = 0; l <= layer; ++l) {
    float nb = 0.f;
    for (int c = 0; c < 16; ++c) nb = fmaxf(nb, fmaf(__ldg(bnd + l * 32 + c), b, __ldg(bnd + l * 32 + 16 + c)));
    nb *= 1.0001f;
    if (!(nb > 0.f) || !isfinite(nb)) nb = 1.f;
    if (l < layer) s_in = stack_scale(nb);
    else s_out = stack_scale(nb);
    b = nb;
  }
}

// x [V] fp32 -> lines [V][64] fp16: channel 0 of both nets = (hi, lo) of x * s_in, everything else 0
__global__ void __launch_bounds__(256) nc_stack_pack_kernel(const float* __restrict__ x, size_t V, const float* bnd,
                                                            const unsigned int* xmax, uint4* __restrict__ lines) {
  float s_in, s_out;
  stack_scales(bnd, xmax, 0, s_in, s_out);
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < V * 8; i += (size_t)gridDim.x * blockDim.x) {
    const size_t v = i >> 3;
    const int q = (int)(i & 7);                  // 16-byte quarter of the line: 0 net0 hi, 2 net0 lo, 4 net1 hi, 6 net1 lo
    uint4 w = make_uint4(0, 0, 0, 0);
    if ((q & 1) == 0) {
      const float f = __ldg(x + v) * s_in;
      const __half h = __float2half_rn(f);
      w.x = (q & 2) ? (uint32_t)__half_as_ushort(__float2half_rn(f - __half2float(h))) : (uint32_t)__half_as_ushort(h);
    }
    lines[i] = w;
  }
}

template <int K, int NETS>
__global__ void __launch_bounds__(384, 1) nc_stack_layer_kernel(const __grid_constant__ NcStackLayerParams p,
                                                                const __grid_constant__ CUtensorMap lmap) {
  constexpr int PAD = K / 2;
  constexpr int WSTAGE = K * kStackWTap;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* wsm = smem + (size_t)p.ring_b * p.unit_b;
  __shared__ __align__(8) uint64_t bfull[kStackRing], bempty[kStackRing], wfull[kStackRing], wempty[kStackRing];

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int per_a = p.KB * p.LB;
  if (warp == 1 && lane == 0) {
    for (int i = 0; i < kStackRing; ++i) {
      mbar_init(&bfull[i], 1);
      mbar_init(&bempty[i], 2);
      mbar_init(&wfull[i], 1);
      mbar_init(&wempty[i], 2);
    }
    fence_barrier_init();
  }
  if (warp == 3 && lane == 0) tma_prefetch_desc(&lmap);
  __syncthreads();

  const int wgi = warpgroup_index();
  if (warp == 3) {
    // ===================== loader: per valid A-tap one block, then k weight stages =====================
    if (lane == 0) {
      const uint32_t box_bytes = (uint32_t)((p.TW + 2 * PAD) * (p.R + 2 * PAD) * 128);
      int ub = 0, uw = 0;
      for (int tile = blockIdx.x; tile < p.tiles; tile += gridDim.x) {
        const int a = tile / per_a, rem = tile - a * per_a;
        const int kb = rem / p.LB, lb = rem - kb * p.LB;
        const int ia = a / p.wA, ja = a - ia * p.wA;
        const int i0 = max(0, PAD - ia), i1 = min(K, p.hA - ia + PAD);
        const int j0 = max(0, PAD - ja), j1 = min(K, p.wA - ja + PAD);
        for (int ti = i0; ti < i1; ++ti)
          for (int tj = j0; tj < j1; ++tj) {
            const int s = ub % p.ring_b;
            mbar_wait(&bempty[s], ((uint32_t)(ub / p.ring_b) & 1u) ^ 1u);
            mbar_expect_tx(&bfull[s], box_bytes);
            tma_load_4d(&lmap, &bfull[s], smem + (size_t)s * p.unit_b, 0, lb * p.TW - PAD, kb * p.R - PAD,
                        (ia + ti - PAD) * p.wA + (ja + tj - PAD));
            ++ub;
            const __half* wsrc = p.wimg + (size_t)(ti * K + tj) * K * K * (kStackWTap / 2);
            for (int tk = 0; tk < K; ++tk, ++uw) {
              const int w = uw % p.ring_w;
              mbar_wait(&wempty[w], ((uint32_t)(uw / p.ring_w) & 1u) ^ 1u);
              mbar_expect_tx(&wfull[w], (uint32_t)WSTAGE);
              bulk_load(&wfull[w], wsm + (size_t)w * WSTAGE, wsrc + (size_t)tk * K * (kStackWTap / 2), (uint32_t)WSTAGE);
            }
          }
      }
    }
  } else if (wgi >= 1) {
    // ===================== MMA + epilogue: warpgroup wg owns MMA rows 64 wg .. 64 wg + 63 =====================
    const int wg = wgi - 1, wl = warp & 3;
    const bool leader = threadIdx.x % 128 == 0;
    const int t = lane & 3;
    const int m0 = wg * 64 + 16 * wl + (lane >> 2);          // fragment rows m0 and m0 + 8
    float s_in, s_out;
    stack_scales(p.bnd, p.xmax, p.layer, s_in, s_out);
    const float inv = p.inv_sw / s_in;
    const uint32_t sbase = smem_u32(smem), wbase = smem_u32(wsm);
    const uint32_t tk_stride = (uint32_t)(p.P * 128);
    int ub = 0, uw = 0;
    for (int tile = blockIdx.x; tile < p.tiles; tile += gridDim.x) {
      const int a = tile / per_a, rem = tile - a * per_a;
      const int kb = rem / p.LB, lb = rem - kb * p.LB;
      const int ia = a / p.wA, ja = a - ia * p.wA;
      const int i0 = max(0, PAD - ia), i1 = min(K, p.hA - ia + PAD);
      const int j0 = max(0, PAD - ja), j1 = min(K, p.wA - ja + PAD);
      float tot[NETS][8];
#pragma unroll
      for (int n = 0; n < NETS; ++n)
#pragma unroll
        for (int i = 0; i < 8; ++i) tot[n][i] = 0.f;
      for (int ti = i0; ti < i1; ++ti)
        for (int tj = j0; tj < j1; ++tj) {
          float da[NETS][16], db[NETS][8];     // per net: [0,8) hi*hi, [8,16) hi*lo ; lo*hi
          const int s = ub % p.ring_b;
          mbar_wait(&bfull[s], (uint32_t)(ub / p.ring_b) & 1u);
          const uint32_t blk = sbase + (uint32_t)(s * p.unit_b) + (uint32_t)(wg * 64 * 128);
          int wprev = -1;
#pragma unroll
          for (int tk = 0; tk < K; ++tk, ++uw) {
            const int w = uw % p.ring_w;
            mbar_wait(&wfull[w], (uint32_t)(uw / p.ring_w) & 1u);
            wgmma_fence();
#pragma unroll
            for (int tl = 0; tl < K; ++tl) {
              // 128-byte granular start, base offset 0: the 128B swizzle is a function of the address bits
              const uint64_t adesc = make_sw128_desc(blk + (uint32_t)tk * tk_stride + (uint32_t)(tl * 128));
              const uint64_t wdesc = make_sw128_desc(wbase + (uint32_t)(w * WSTAGE + tl * kStackWTap));
              const uint32_t acc = (tk > 0 || tl > 0) ? 1u : 0u;
#pragma unroll
              for (int n = 0; n < NETS; ++n) {
                wgmma_f16<32>(da[n], adesc + 2 * (n * 2), wdesc + 2 * n, acc);       // hi*hi | hi*lo
                wgmma_f16<16>(db[n], adesc + 2 * (n * 2 + 1), wdesc + 2 * n, acc);   // lo*hi
              }
            }
            wgmma_commit();
            if (tk > 0) {
              wgmma_wait<1>();                      // the MMAs of row tk - 1 have read their weight stage
              mbar_arrive_if(&wempty[wprev], leader);
            }
            wprev = w;
          }
          wgmma_wait<0>();
#pragma unroll
          for (int n = 0; n < NETS; ++n) {
            wgmma_fence_regs<16>(da[n]);
            wgmma_fence_regs<8>(db[n]);
          }
          mbar_arrive_if(&wempty[wprev], leader);
          mbar_arrive_if(&bempty[s], leader);
          ++ub;
#pragma unroll
          for (int n = 0; n < NETS; ++n)
#pragma unroll
            for (int i = 0; i < 8; ++i) tot[n][i] += (db[n][i] + da[n][8 + i]) + da[n][i];
        }
      // ---- epilogue ----
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int m = m0 + 8 * h;
        const int kk = m / p.P, ll = m - kk * p.P;
        const int kq = kb * p.R + kk, lq = lb * p.TW + ll;
        if (kk < p.R && ll < p.TW && kq < p.hB && lq < p.wB) {
          const size_t v = (size_t)a * p.nB + (size_t)kq * p.wB + lq;
          if (p.last) {
            if (t == 0) {                       // channel 0 = fragment column 0 of quad lane 0
              float o = 0.f;
#pragma unroll
              for (int n = 0; n < NETS; ++n) o += fmaxf(fmaf(tot[n][2 * h], inv, __ldg(p.bias)), 0.f);
              p.out[v] = o;
            }
          } else {
            uint32_t* line = reinterpret_cast<uint32_t*>(p.out_lines + v * 64);
#pragma unroll
            for (int n = 0; n < NETS; ++n)
#pragma unroll
              for (int j = 0; j < 2; ++j) {
                const int c = 8 * j + 2 * t;      // channels c, c + 1
                float hv[2];
#pragma unroll
                for (int e = 0; e < 2; ++e)
                  hv[e] = fmaxf(fmaf(tot[n][4 * j + 2 * h + e], inv, __ldg(p.bias + c + e)), 0.f) * s_out;
                const __half2 hi = __floats2half2_rn(hv[0], hv[1]);
                const float2 hf = __half22float2(hi);
                const __half2 lo = __floats2half2_rn(hv[0] - hf.x, hv[1] - hf.y);
                line[(n * 32 + c) >> 1] = *reinterpret_cast<const uint32_t*>(&hi);
                line[(n * 32 + 16 + c) >> 1] = *reinterpret_cast<const uint32_t*>(&lo);
              }
          }
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
static float stack_pow2_scale(float maxabs, float target_hi) {   // power of two s: maxabs * s in [target_hi/2, target_hi)
  if (!(maxabs > 0.f) || !isfinite(maxabs)) return 1.f;
  int e, et;
  frexpf(maxabs, &e);
  frexpf(target_hi, &et);
  return ldexpf(1.f, et - 1 - e);
}

static inline size_t stack_sw128_index(int n, int k) { return (size_t)n * 64 + ((((k >> 3) ^ (n & 7)) << 3) | (k & 7)); }

void nc_stack_release(NcStackWeights& S) {
  if (S.blob) cudaFree(S.blob);
  S = NcStackWeights();
}

int nc_stack_pack(int n_layers, const int* ks, const int* chans, const float* const* weights, const float* const* biases,
                  int symmetric, NcStackWeights& S) {
  P2P_REQUIRE(n_layers >= 1 && n_layers <= kNcStackMaxLayers, "n_layers must be in 1..16");
  for (int l = 0; l < n_layers; ++l) {
    P2P_REQUIRE(ks[l] == 3 || ks[l] == 5, "kernel sizes must be 3 or 5");
    P2P_REQUIRE(chans[l] >= 1 && chans[l] <= 16, "channels must be in 1..16");
    P2P_REQUIRE(weights[l] != nullptr && biases[l] != nullptr, "null weight pointer");
  }
  P2P_REQUIRE(chans[n_layers - 1] == 1, "the last layer must have 1 output channel");
  std::vector<size_t> off(n_layers);
  size_t total = 0;
  for (int l = 0; l < n_layers; ++l) {
    off[l] = total;
    const size_t k2 = (size_t)ks[l] * ks[l];
    total += align_up(k2 * k2 * kStackWTap, 1024);
  }
  const size_t img_bytes = total;
  total += (size_t)n_layers * 16 * 4 + (size_t)n_layers * 32 * 4;
  std::vector<char> host(total, 0);
  std::vector<float> bias(n_layers * 16, 0.f), bnd(n_layers * 32, 0.f);
  NcStackWeights W;
  W.n_layers = n_layers;
  W.symmetric = symmetric ? 1 : 0;
  for (int l = 0; l < n_layers; ++l) {
    const int k = ks[l], co_n = chans[l], ci_n = l == 0 ? 1 : chans[l - 1];
    const float* w = weights[l];   // reference layout [k][Cout][Cin][k][k][k]
    auto at = [&](int co, int ci, int a1, int a2, int b1, int b2) {
      return w[((((size_t)a1 * co_n + co) * ci_n + ci) * k + a2) * k * k + (size_t)b1 * k + b2];
    };
    float m = 0.f;
    for (size_t i = 0; i < (size_t)k * k * k * k * co_n * ci_n; ++i) m = fmaxf(m, fabsf(w[i]));
    const float s = stack_pow2_scale(m, 1024.f);
    W.ks[l] = k;
    W.chans[l] = co_n;
    W.inv_sw[l] = 1.f / s;
    __half* img = reinterpret_cast<__half*>(host.data() + off[l]);
    for (int co = 0; co < co_n; ++co) {
      float sum = 0.f;
      for (int a1 = 0; a1 < k; ++a1)
        for (int a2 = 0; a2 < k; ++a2)
          for (int b1 = 0; b1 < k; ++b1)
            for (int b2 = 0; b2 < k; ++b2) {
              __half* tap = img + ((size_t)((a1 * k + a2) * k + b1) * k + b2) * (kStackWTap / 2);
              for (int ci = 0; ci < ci_n; ++ci) {
                sum += fabsf(at(co, ci, a1, a2, b1, b2));
                for (int net = 0; net < 1 + W.symmetric; ++net) {
                  // net 1: the A and B tap axes swapped
                  const float v = (net == 0 ? at(co, ci, a1, a2, b1, b2) : at(co, ci, b1, b2, a1, a2)) * s;
                  const __half hi = __float2half_rn(v), lo = __float2half_rn(v - __half2float(hi));
                  tap[stack_sw128_index(co, net * 16 + ci)] = hi;
                  tap[stack_sw128_index(16 + co, net * 16 + ci)] = lo;
                }
              }
            }
      bias[l * 16 + co] = biases[l][co];
      bnd[l * 32 + co] = sum * 1.0001f;
      bnd[l * 32 + 16 + co] = fabsf(biases[l][co]);
    }
  }
  memcpy(host.data() + img_bytes, bias.data(), bias.size() * 4);
  memcpy(host.data() + img_bytes + bias.size() * 4, bnd.data(), bnd.size() * 4);
  if (cudaMalloc(&W.blob, total) != cudaSuccess) {
    cudaGetLastError();
    set_last_error("out of device memory packing the NeighConsensus stack weights");
    return -3;
  }
  if (cudaMemcpy(W.blob, host.data(), total, cudaMemcpyHostToDevice) != cudaSuccess) {
    cudaFree(W.blob);
    set_last_error("copying the NeighConsensus stack weights failed");
    return -2;
  }
  for (int l = 0; l < n_layers; ++l) {
    W.img[l] = reinterpret_cast<const __half*>(W.blob + off[l]);
    W.bias[l] = reinterpret_cast<const float*>(W.blob + img_bytes) + l * 16;
  }
  W.bnd = reinterpret_cast<const float*>(W.blob + img_bytes + bias.size() * 4);
  nc_stack_release(S);
  S = W;
  return 0;
}

size_t nc_stack_scratch_bytes(size_t V) { return 2 * V * 128 + 4096; }

// B-grid tiling: the TW with the fewest tiles (R rows of TW columns, pitch TW + 2p, filling 128 MMA rows) whose block
// buffer fits twice in shared memory beside the weight ring (wide B grids take narrower tiles)
static void stack_geometry(int hB, int wB, int k, int wbytes, NcStackLayerParams& p) {
  const int pad = k / 2;
  long long best = -1;
  for (int tw = wB < 128 ? wB : 128; tw >= 1; --tw) {
    const int P = tw + 2 * pad, R = (128 - tw) / P + 1;
    const int lines_box = (R + 2 * pad) * P, lines_read = 128 + 2 * pad * P + 2 * pad;
    const int unit = (int)align_up((size_t)(lines_box > lines_read ? lines_box : lines_read) * 128, 1024);
    if (2 * unit + wbytes > kStackSmemBudget) continue;
    const long long n = (long long)cdiv(wB, tw) * cdiv(hB, R);
    if (best < 0 || n < best) {
      best = n;
      p.TW = tw; p.R = R; p.P = P; p.unit_b = unit;
    }
  }
  p.KB = cdiv(hB, p.R);
  p.LB = cdiv(wB, p.TW);
}

template <int K, int NETS>
static int launch_stack_layer(const NcStackLayerParams& p, const CUtensorMap& m, int grid, int smem, cudaStream_t st) {
  auto kern = nc_stack_layer_kernel<K, NETS>;
  P2P_ENSURE_SMEM(kern, smem);
  kern<<<grid, 384, smem, st>>>(p, m);
  P2P_LAUNCH_OK();
  return 0;
}

int launch_nc_stack(const float* x, int hA, int wA, int hB, int wB, const NcStackWeights& W, const unsigned int* xmax,
                    __half* scratch, float* out, int num_sms, cudaStream_t st) {
  const int nA = hA * wA, nB = hB * wB;
  const size_t V = (size_t)nA * nB;
  __half* buf[2] = {scratch, scratch + V * 64};
  {
    const size_t n = V * 8;
    const int blocks = (int)((n + 255) / 256 < 4096 ? (n + 255) / 256 : 4096);
    nc_stack_pack_kernel<<<blocks, 256, 0, st>>>(x, V, W.bnd, xmax, reinterpret_cast<uint4*>(buf[0]));
    P2P_LAUNCH_OK();
  }
  for (int l = 0; l < W.n_layers; ++l) {
    NcStackLayerParams p;
    memset(&p, 0, sizeof(p));
    p.hA = hA; p.wA = wA; p.hB = hB; p.wB = wB; p.nA = nA; p.nB = nB;
    p.k = W.ks[l]; p.p = p.k / 2;
    p.cout = W.chans[l];
    p.layer = l;
    p.last = l == W.n_layers - 1;
    const int wstage = p.k * kStackWTap;
    p.ring_w = p.k == 3 ? 6 : 4;
    stack_geometry(hB, wB, p.k, p.ring_w * wstage, p);
    const long long tiles = (long long)nA * p.KB * p.LB;
    P2P_REQUIRE(tiles < (1ll << 30), "NeighConsensus stack: 4D volume too large");
    p.tiles = (int)tiles;
    p.ring_b = (kStackSmemBudget - p.ring_w * wstage) / p.unit_b;
    if (p.ring_b > kStackRing) p.ring_b = kStackRing;
    P2P_REQUIRE(p.ring_b >= 2, "NeighConsensus stack: block buffer does not fit in shared memory");
    p.wimg = W.img[l];
    p.bias = W.bias[l];
    p.bnd = W.bnd;
    p.inv_sw = W.inv_sw[l];
    p.xmax = xmax;
    p.out_lines = buf[(l + 1) & 1];
    p.out = out;
    CUtensorMap lmap;
    const uint64_t dims[4] = {64, (uint64_t)wB, (uint64_t)hB, (uint64_t)nA};
    const uint64_t strides[3] = {128, (uint64_t)wB * 128, (uint64_t)nB * 128};
    const uint32_t box[4] = {64, (uint32_t)(p.TW + 2 * p.p), (uint32_t)(p.R + 2 * p.p), 1};
    int rc = make_tmap_fp16(&lmap, buf[l & 1], 4, dims, strides, box);
    if (rc) return rc;
    const int smem = p.ring_b * p.unit_b + p.ring_w * wstage + 1024;
    const int grid = p.tiles < num_sms ? p.tiles : num_sms;
    if (p.k == 3) rc = W.symmetric ? launch_stack_layer<3, 2>(p, lmap, grid, smem, st) : launch_stack_layer<3, 1>(p, lmap, grid, smem, st);
    else rc = W.symmetric ? launch_stack_layer<5, 2>(p, lmap, grid, smem, st) : launch_stack_layer<5, 1>(p, lmap, grid, smem, st);
    if (rc) return rc;
  }
  return 0;
}

}  // namespace p2p
