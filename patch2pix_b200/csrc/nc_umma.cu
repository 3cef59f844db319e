// NeighConsensus (symmetric 2-layer Conv4d 1 -> 16 -> 1, k = 3, ReLU after each layer) on the Hopper tensor cores (wgmma).
//
// Reference semantics (file:line relative to the reference repo):
//   NeighConsensus.forward   networks/ncn/model.py:145-155   conv(x) + conv(x^T)^T, shared weights
//   Conv4d / conv4d          networks/ncn/conv4d.py:12-130   true 4D cross-correlation, zero "same" padding
//
// conv(x) + conv(x^T)^T equals two independent nets on the SAME input, the second with tap axes (a,b) <-> (d,e)
// swapped (api.cu packs both: w1p / w2p [81 taps][32 = 16 ch of net 0 | 16 ch of net 1]).
//
// Both layers are skinny GEMMs on wgmma; nothing but x, the hidden tensor and the partial maps touches HBM and no
// FMA-pipe inner loop is left:
//
//   pad/split x -> xp: zero-haloed copy of x, every element already scaled and split into an fp16 (hi, lo) pair packed
//             in one 32-bit word, so layer 1 needs neither bounds logic nor conversions.
//   layer 1   rows = 128 consecutive B cells of one A cell, K = 81 taps (padded to 128), N = 32 channels (both nets).
//             Producer warps build the im2col operand in shared memory (ld.shared + prmt + st.shared only) from the
//             tile's 9 neighbour blocks, which one thread stages with bulk copies (cp.async.bulk).
//             Epilogue: + bias, ReLU, re-scale, fp16 hi/lo split -> hidden[cell][64 fp16] =
//             [net0 hi 16 | net0 lo 16 | net1 hi 16 | net1 lo 16] (one 128-byte line per cell).
//   layer 2   16 -> 1 channels would be an N = 1 GEMM.  Instead, per hidden cell a' and per net, the 9 PARTIAL maps
//             P_(ta,tb)[a'][b] = sum over the 9 B-taps and 16 channels are one GEMM with K = 9 x 16 = 144, N = 9
//             (padded to 16).  The A operand of a B-tap is the tile's block of hidden lines SHIFTED by the tap offset:
//             the block (with its zero halo, courtesy of TMA out-of-bounds fill) is loaded ONCE per tile and every tap
//             only moves the start address of the shared-memory descriptor -- there are no producer warps at all.
//   combine   out[a][b] = sum_net relu(b2 + sum_(ta,tb) P_(ta,tb)[a + (ta-1, tb-1)][b])  (fixed summation order:
//             deterministic), fused with the row/column maxima of the MutualMatching that follows.
//
// Precision: fp16 hi/lo operand pairs, three products per term (lo*hi + hi*lo + hi*hi, fp32 accumulate in registers, each
// product kind in its own accumulator so the chains are short and independent): products good to ~2^-22, i.e.
// fp32-grade.  Activations are scaled by powers of two derived ON THE DEVICE from max|x| (and from a weight-norm bound
// for the hidden tensor), so any input range is safe in fp16.
//
// Warp-specialised persistent kernels (loader thread, two consumer warpgroups that issue the MMAs and run the epilogue
// on the accumulator fragments, producer warps in layer 1) with mbarrier rings.
#include <math.h>

#include <type_traits>
#include <vector>

#include "kernels.h"
#include "umma_gemm.h"
#include "umma_ptx.cuh"

namespace p2p {

constexpr int kNcAtom = 128 * 128;   // bytes of one [128 rows x 64 fp16] swizzled operand atom

struct NcParams {
  int hA, wA, hB, wB, nA, nB;
  long long V;                 // nA * nB cells
  const float* x;              // [V] input (after the first MutualMatching)
  const unsigned int* xmax;    // device: float bits of max |x|
  uint32_t* xp;                // [(hA+2)(wA+2)][hB+2][WP] zero-haloed (hi | lo << 16) fp16 pairs of x * sx
  __half* hidden;              // [V][64]
  float* partial;              // [2 nets][9][V]
  const __half* wimg;          // weight operand image, laid out exactly as in shared memory
  const float* b1p;            // [32]
  float wsum1, b1max;          // max_c sum_taps |w1|, max |b1|: bound of the hidden activations
  float inv_sw1, inv_sw2;      // 1 / (power-of-two weight scales)
  int tiles;
  int WP;                      // padded row pitch of xp (multiple of 4 words)
  int l1_bufs;                 // layer-1 staging buffers: 2 (copies of tile i+1 overlap tile i) or 1 (wide B grids)
  // layer 2 tiling: tile = R rows x TW columns of one A cell's B grid, enumerated with pitch P lines
  int TW, R, P, KB, LB;        // KB x LB tiles per A cell
  int copies;                  // 1: one haloed block per tile (pitch TW + 2); 3: one block per column tap (pitch TW)
  int ring, unit_bytes;        // ring of block buffers in shared memory
  int l2_ctas;                 // CTAs of layer 2 per SM (1 or 2)
};

// Power-of-two activation scales: max|x| * sx and (hidden bound) * sh land in [2048, 4096).
__device__ __forceinline__ void nc_scales(const NcParams& p, float& sx, float& sh) {
  float xmax = __uint_as_float(__ldg(p.xmax));
  if (!(xmax > 0.f) || !isfinite(xmax)) xmax = 1.f;
  int e;
  frexpf(xmax, &e);
  sx = ldexpf(1.f, min(12 - e, 60));
  float hb = fmaf(p.wsum1, xmax, p.b1max);
  if (!(hb > 0.f) || !isfinite(hb)) hb = 1.f;
  frexpf(hb, &e);
  sh = ldexpf(1.f, min(12 - e, 60));
}

// exact n / d for 0 <= n < 2^22 with inv = 1.f / d (the quotient of n + 0.5 is at least 0.5 / d away from an integer)
__device__ __forceinline__ int fast_div(int n, float inv) { return __float2int_rz(((float)n + 0.5f) * inv); }

__device__ __forceinline__ uint32_t lds_u32(uint32_t addr) {
  uint32_t v;
  asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(addr));
  return v;
}
__device__ __forceinline__ void sts_v4(uint32_t addr, uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
  asm volatile("st.shared.v4.u32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(a), "r"(b), "r"(c), "r"(d) : "memory");
}

// ------------------------------------------------------------------------------------------------
// pad / split: x [nA][hB][wB] fp32 -> xp [(hA+2)(wA+2)][hB+2][WP] words (fp16 hi | fp16 lo << 16) of x * sx, zero halo.
// One block per padded A cell.
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) nc_pad_split_kernel(const __grid_constant__ NcParams p) {
  const int pa = blockIdx.x;
  const int pi = pa / (p.wA + 2), pj = pa - pi * (p.wA + 2);
  const bool inside = pi >= 1 && pi <= p.hA && pj >= 1 && pj <= p.wA;
  float sx, sh;
  nc_scales(p, sx, sh);
  const int n = (p.hB + 2) * p.WP;
  uint32_t* dst = p.xp + (size_t)pa * n;
  const float* src = inside ? p.x + (size_t)((pi - 1) * p.wA + (pj - 1)) * p.nB : p.x;
  const float inv = 1.f / (float)p.WP;
  for (int i = threadIdx.x; i < n; i += 256) {
    const int kp = fast_div(i, inv), lp = i - kp * p.WP;
    uint32_t w = 0;
    if (inside && kp >= 1 && kp <= p.hB && lp >= 1 && lp <= p.wB) {
      const float v = src[(kp - 1) * p.wB + (lp - 1)] * sx;
      const __half h = __float2half_rn(v), l = __float2half_rn(v - __half2float(h));
      w = (uint32_t)__half_as_ushort(h) | ((uint32_t)__half_as_ushort(l) << 16);
    }
    dst[i] = w;
  }
}

// ------------------------------------------------------------------------------------------------
// layer 1.  Tile = (A cell a, 128 consecutive B cells).  The B rows of the 9 A-neighbours the tile touches are staged
// from xp with 9 bulk copies by one thread (double-buffered: tile i+1 is in flight while tile i is built), so a tap is
// a plain `ld.shared [row base + tk*pitch + tl]` with no validity logic.  Eight producer warps (two threads per tile
// row, each half of the 11 tap chunks) pack the (hi, lo) words into the swizzled operand chunks.
// Two consumer warpgroups (tile rows 0..63 and 64..127) run the MMAs: the three products of the hi/lo split (lo*hi,
// hi*lo, hi*hi) accumulate in SEPARATE register accumulators -- a_hi x [w_hi | w_lo] (N = 64) gives hi*hi and hi*lo,
// a_lo x w_hi (N = 32) gives lo*hi -- and are summed by the epilogue, which works on the accumulator fragments directly.
// 640 threads (warp 3 loader, warps 4..11 MMA + epilogue, 12..19 producers), 1 CTA per SM, 4 x 32 KB operand stages.
// ------------------------------------------------------------------------------------------------
constexpr int kL1Stages = 4;
constexpr int kL1Threads = 640, kL1ProducerWarps = 8;

__host__ __device__ inline int nc_l1_rows(int wB) { return 127 / wB + 4; }      // padded B rows a tile can touch

__global__ void __launch_bounds__(kL1Threads, 1) nc_l1_umma_kernel(const __grid_constant__ NcParams p,
                                                                  const __grid_constant__ CUtensorMap hstore) {
  constexpr int STAGE_BYTES = 2 * kNcAtom;         // A_hi + A_lo of one atom
  constexpr int WATOM = 64 * 128;                  // weight image of one atom: rows 0..31 w_hi, 32..63 w_lo
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* wsm = smem + kL1Stages * STAGE_BYTES;                          // [atom][hi|lo] weight images, 16 KB
  uint8_t* hst = wsm + 2 * WATOM;                                         // 2 x 16 KB staging of finished hidden tiles
  uint8_t* xs = hst + 2 * kNcAtom;                                        // [bufs][9][rows][pitch] words
  __shared__ __align__(8) uint64_t full_bar[kL1Stages];
  __shared__ __align__(8) uint64_t empty_bar[kL1Stages];
  __shared__ __align__(8) uint64_t xfull_bar[2];
  __shared__ __align__(8) uint64_t xempty_bar[2];

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tiles = p.tiles;
  const int TB = (p.nB + 127) >> 7;
  const int NR = nc_l1_rows(p.wB);
  const uint32_t NRB = (uint32_t)(NR * p.WP * 4);                         // bytes of one neighbour block
  const float inv_tb = 1.f / (float)TB, inv_wb = 1.f / (float)p.wB;
  const int nbuf = p.l1_bufs;

  for (int i = threadIdx.x; i < kL1Stages * STAGE_BYTES / 16; i += kL1Threads) reinterpret_cast<uint4*>(smem)[i] = make_uint4(0, 0, 0, 0);
  for (int i = threadIdx.x; i < 2 * WATOM / 16; i += kL1Threads)
    reinterpret_cast<uint4*>(wsm)[i] = __ldg(reinterpret_cast<const uint4*>(p.wimg) + i);
  if (warp == 1 && lane == 0) {
    for (int i = 0; i < kL1Stages; ++i) {
      mbar_init(&full_bar[i], kL1ProducerWarps);
      mbar_init(&empty_bar[i], 2);
    }
    for (int i = 0; i < 2; ++i) {
      mbar_init(&xfull_bar[i], 1);
      mbar_init(&xempty_bar[i], kL1ProducerWarps);
    }
    fence_barrier_init();
  }
  fence_proxy_async();
  __syncthreads();

  const int wgi = warpgroup_index();
  if (wgi == 1 || wgi == 2) {
    // ===================== MMA + epilogue: warpgroup wg owns tile rows 64 wg .. 64 wg + 63 =====================
    const int wg = wgi - 1, wl = warp & 3;
    const bool leader = threadIdx.x % 128 == 0;
    const int t = lane & 3;
    const int r0 = wg * 64 + 16 * wl + (lane >> 2);          // fragment rows r0 and r0 + 8
    float sx, sh;
    nc_scales(p, sx, sh);
    const float inv = p.inv_sw1 / sx;
    const uint32_t sbase = smem_u32(smem), wbase = smem_u32(wsm);
    int it = 0, tl = 0;
    for (int tile = blockIdx.x; tile < tiles; tile += gridDim.x, ++tl) {
      float d64[32], d32[16];                                // [0,32) hi*hi | [32,64) hi*lo ; lo*hi
      int st[2];
#pragma unroll
      for (int atom = 0; atom < 2; ++atom, ++it) {
        const int s = it % kL1Stages;
        st[atom] = s;
        mbar_wait(&full_bar[s], (uint32_t)(it / kL1Stages) & 1u);
        const uint32_t sa = sbase + (uint32_t)(s * STAGE_BYTES) + (uint32_t)(wg * 8192);
        const uint64_t a_hi = make_sw128_desc(sa), a_lo = make_sw128_desc(sa + kNcAtom);
        const uint64_t w = make_sw128_desc(wbase + (uint32_t)(atom * WATOM));     // rows 0..31 w_hi, 32..63 w_lo
        constexpr int nk0 = 4, nk1 = 2;             // taps 64..80 live in the first two K16 slices of atom 1
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < nk0; ++kk) {
          if (atom == 1 && kk >= nk1) break;
          const uint32_t acc = (atom > 0 || kk > 0) ? 1u : 0u;
          wgmma_f16<64>(d64, a_hi + 2 * kk, w + 2 * kk, acc);      // hi*hi | hi*lo
          wgmma_f16<32>(d32, a_lo + 2 * kk, w + 2 * kk, acc);      // lo*hi
        }
        wgmma_commit();
      }
      wgmma_wait<0>();
      wgmma_fence_regs<32>(d64);
      wgmma_fence_regs<16>(d32);
      mbar_arrive_if(&empty_bar[st[0]], leader);
      mbar_arrive_if(&empty_bar[st[1]], leader);
      const int a = fast_div(tile, inv_tb), b0 = (tile - a * TB) << 7;
      // The tile's 128 hidden lines are contiguous in global memory.  They go through a swizzled shared staging
      // buffer and leave with ONE tensor-map store per tile.  Rows past the end of the B grid are clipped by the
      // tensor map.
      uint8_t* sb = hst + (size_t)(tl & 1) * kNcAtom;
      if (threadIdx.x == 128) bulk_wait_group_read<1>();        // the store of tile tl-2 has finished reading this buffer
      asm volatile("bar.sync 2, 256;" ::: "memory");
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int row = r0 + 8 * h;
        if (b0 + row < p.nB) {
          const uint32_t so = smem_u32(sb) + (uint32_t)(row * 128);
          const uint32_t sw = (uint32_t)(row & 7);
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const int c = 8 * j + 2 * t;                           // channels c, c + 1: net c / 16
            float hv[2];
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int i = 4 * j + 2 * h + e;
              const float acc = (d32[i] + d64[16 + i]) + d64[i];   // (lo*hi + hi*lo) + hi*hi
              hv[e] = fmaxf(fmaf(acc, inv, __ldg(p.b1p + c + e)), 0.f) * sh;
            }
            const __half2 hi = __floats2half2_rn(hv[0], hv[1]);
            const float2 hf = __half22float2(hi);
            const __half2 lo = __floats2half2_rn(hv[0] - hf.x, hv[1] - hf.y);
            const int idx = (c >> 4) * 32 + (c & 15);                 // [net][hi 16 | lo 16]
            const uint32_t chi = (uint32_t)(idx >> 3), clo = chi + 2, wi = (uint32_t)((idx & 7) * 2);
            asm volatile("st.shared.b32 [%0], %1;" ::"r"(so + ((chi ^ sw) << 4) + wi), "r"(*reinterpret_cast<const uint32_t*>(&hi)) : "memory");
            asm volatile("st.shared.b32 [%0], %1;" ::"r"(so + ((clo ^ sw) << 4) + wi), "r"(*reinterpret_cast<const uint32_t*>(&lo)) : "memory");
          }
        }
      }
      fence_proxy_async();
      asm volatile("bar.sync 2, 256;" ::: "memory");
      if (threadIdx.x == 128) {
        tma_store_3d(&hstore, sb, 0, b0, a);
        bulk_commit_group();
      }
    }
    if (threadIdx.x == 128) bulk_wait_group_read<0>();
  } else if (warp == 3) {
    // ===================== loader: 9 bulk copies per tile =====================
    if (lane == 0) {
      int tl = 0;
      for (int tile = blockIdx.x; tile < tiles; tile += gridDim.x, ++tl) {
        const int buf = nbuf == 2 ? (tl & 1) : 0;
        mbar_wait(&xempty_bar[buf], ((uint32_t)(nbuf == 2 ? (tl >> 1) : tl) & 1u) ^ 1u);
        const int a = fast_div(tile, inv_tb), b0 = (tile - a * TB) << 7;
        const int ia = a / p.wA, ja = a - ia * p.wA;
        const int k0 = fast_div(b0, inv_wb);                          // padded row k0 = unpadded row k0 - 1
        mbar_expect_tx(&xfull_bar[buf], 9u * NRB);
        uint8_t* dst = xs + (size_t)buf * 9 * NRB;
#pragma unroll
        for (int d = 0; d < 9; ++d) {
          const int pa = (ia + d / 3) * (p.wA + 2) + ja + d % 3;
          bulk_load(&xfull_bar[buf], dst + (size_t)d * NRB, p.xp + ((size_t)pa * (p.hB + 2) + k0) * p.WP, NRB);
        }
      }
    }
  } else if (warp >= 12) {
    // ===================== producers: 256 threads = 128 tile rows x 2 chunk halves =====================
    const int ptid = threadIdx.x - 384;
    const int r = ptid & 127;
    const int qh = ptid >> 7;          // warp-uniform: quarters 2 qh and 2 qh + 1 (chunks Q, Q + 4 of atom 0, Q of atom 1)
    const uint32_t sw = (uint32_t)(r & 7);
    const uint32_t otk = (uint32_t)(p.WP * 4);
    int it = 0, tl = 0;
    for (int tile = blockIdx.x; tile < tiles; tile += gridDim.x, ++tl) {
      const int buf = nbuf == 2 ? (tl & 1) : 0;
      const int a = fast_div(tile, inv_tb), b0 = (tile - a * TB) << 7;
      const int b = b0 + r;
      const bool rv = b < p.nB;                                // rows past the end of the B grid are not built: their
      const int k = fast_div(b, inv_wb), l = b - k * p.wB;     // operand rows keep stale data and the epilogue skips them
      const int k0 = fast_div(b0, inv_wb);
      // shared address of the (tk, tl) = (0, 0) tap of A-neighbour 0: tap (d, tk, tl) is at + d*NRB + tk*otk + tl*4
      const uint32_t base = smem_u32(xs) + (uint32_t)buf * 9u * NRB + (uint32_t)(((k - k0) * p.WP + l) * 4);
      mbar_wait(&xfull_bar[buf], (uint32_t)(nbuf == 2 ? (tl >> 1) : tl) & 1u);
      auto chunk = [&](auto ATOM, auto CH, uint32_t st) {
        constexpr int atom = decltype(ATOM)::value, c = decltype(CH)::value;
        uint32_t w[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          constexpr int t0 = (atom * 8 + c) * 8;
          const int t = t0 + i;                                  // compile-time after unrolling
          w[i] = 0u;
          if (t < 81) {
            const int d = t / 9, tk = (t / 3) % 3, tl2 = t % 3;
            w[i] = lds_u32(base + (uint32_t)d * NRB + (uint32_t)tk * otk + (uint32_t)(tl2 * 4));
          }
        }
        const uint32_t o = st + ((((uint32_t)c) ^ sw) << 4);
        sts_v4(o, __byte_perm(w[0], w[1], 0x5410), __byte_perm(w[2], w[3], 0x5410), __byte_perm(w[4], w[5], 0x5410),
               __byte_perm(w[6], w[7], 0x5410));
        sts_v4(o + kNcAtom, __byte_perm(w[0], w[1], 0x7632), __byte_perm(w[2], w[3], 0x7632),
               __byte_perm(w[4], w[5], 0x7632), __byte_perm(w[6], w[7], 0x7632));
      };
      auto build = [&](auto QH) {
        constexpr int Q0 = 2 * decltype(QH)::value, Q1 = Q0 + 1;
        {   // atom 0: chunks Q, Q + 4 of both quarters
          const int s = it % kL1Stages;
          mbar_wait(&empty_bar[s], ((uint32_t)(it / kL1Stages) & 1u) ^ 1u);
          const uint32_t st = smem_u32(smem) + (uint32_t)(s * STAGE_BYTES + r * 128);
          if (rv) {
            chunk(std::integral_constant<int, 0>{}, std::integral_constant<int, Q0>{}, st);
            chunk(std::integral_constant<int, 0>{}, std::integral_constant<int, Q0 + 4>{}, st);
            chunk(std::integral_constant<int, 0>{}, std::integral_constant<int, Q1>{}, st);
            chunk(std::integral_constant<int, 0>{}, std::integral_constant<int, Q1 + 4>{}, st);
          }
          fence_proxy_async();
          __syncwarp();
          if (lane == 0) mbar_arrive(&full_bar[s]);
          ++it;
        }
        {   // atom 1: chunk Q (taps 64 + 8Q ..; Q = 3 has nothing to write, chunks 3..7 stay zero)
          const int s = it % kL1Stages;
          mbar_wait(&empty_bar[s], ((uint32_t)(it / kL1Stages) & 1u) ^ 1u);
          const uint32_t st = smem_u32(smem) + (uint32_t)(s * STAGE_BYTES + r * 128);
          if (rv) {
            chunk(std::integral_constant<int, 1>{}, std::integral_constant<int, Q0>{}, st);
            if (Q1 < 3) chunk(std::integral_constant<int, 1>{}, std::integral_constant<int, (Q1 < 3 ? Q1 : 0)>{}, st);
          }
          fence_proxy_async();
          __syncwarp();
          if (lane == 0) mbar_arrive(&full_bar[s]);
          ++it;
        }
      };
      if (qh == 0) build(std::integral_constant<int, 0>{});
      else build(std::integral_constant<int, 1>{});
      __syncwarp();
      if (lane == 0) mbar_arrive(&xempty_bar[buf]);            // this warp's reads of the staging buffer are done
    }
  }
}

// ------------------------------------------------------------------------------------------------
// layer 2.  Tile = R rows x TW columns of the B grid of one hidden cell a', both nets, enumerated as MMA rows
// m = kk * P + ll (pitch P lines).  A tensor-map load brings the tile's block of 128-byte hidden lines -- rows
// k0-1 .. k0+R, zero-filled outside the grid -- into shared memory in the 128B-swizzled layout wgmma reads, and the
// A operand of B-tap (tk, tl) is simply that block starting (tk * P + tl) lines further on:
//   copies = 1   the block carries its column halo (box TW + 2 wide, P = TW + 2): one load per tile; the two MMA rows
//                per tile row that fall on the halo are junk and skipped by the epilogue.
//   copies = 3   one block per column tap tl, loaded with the column origin shifted by tl - 1 (P = TW): no junk rows,
//                3 loads per tile (wins when TW + 2 would waste too many of the 128 MMA rows, e.g. wB = 64).
// Tap starts are 128-byte granular, not 1024-byte aligned.  The 128B swizzle -- of TMA writes and of tensor-core
// operand reads alike -- is a pure function of the shared-memory ADDRESS bits (chunk ^= address bits 7..9), so a
// descriptor that starts mid-pattern reads consistently with its "base offset" field left 0.
// Per tap and net: a_hi x [w_hi | w_lo] (one N = 32 MMA gives hi*hi and hi*lo) and a_lo x w_hi (N = 16): four
// independent accumulator chains per tile, summed by the epilogue.
// 384 threads (warp 3 loader, warps 4..11 = two consumer warpgroups, MMA + epilogue); ring of block buffers; two CTAs
// per SM when the ring fits twice, so that one CTA's epilogue overlaps the other's MMAs.
// ------------------------------------------------------------------------------------------------
constexpr int kL2MaxRing = 8;
constexpr int kL2WTap = 32 * 128;     // weight image per B-tap: rows 0..15 w_hi (9 used), 16..31 w_lo; K16 slice = net

template <int COPIES, int CTAS>
__global__ void __launch_bounds__(384, CTAS) nc_l2_umma_kernel(const __grid_constant__ NcParams p,
                                                            const __grid_constant__ CUtensorMap hmap) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* wsm = smem + (size_t)p.ring * p.unit_bytes;      // [9 taps][32 rows][64] weight images, 36 KB
  __shared__ __align__(8) uint64_t full_bar[kL2MaxRing];
  __shared__ __align__(8) uint64_t empty_bar[kL2MaxRing];

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tiles = p.tiles, ring = p.ring;
  constexpr int copies = COPIES;
  const int per_a = p.KB * p.LB;
  const float inv_pa = 1.f / (float)per_a, inv_lb = 1.f / (float)p.LB;

  for (int i = threadIdx.x; i < ring * p.unit_bytes / 16; i += 384) reinterpret_cast<uint4*>(smem)[i] = make_uint4(0, 0, 0, 0);
  for (int i = threadIdx.x; i < 9 * kL2WTap / 16; i += 384)
    reinterpret_cast<uint4*>(wsm)[i] = __ldg(reinterpret_cast<const uint4*>(p.wimg) + i);
  if (warp == 1 && lane == 0) {
    for (int i = 0; i < kL2MaxRing; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 2);
    }
    fence_barrier_init();
  }
  if (warp == 3 && lane == 0) tma_prefetch_desc(&hmap);
  fence_proxy_async();
  __syncthreads();

  const int wgi = warpgroup_index();
  if (warp == 3) {
    // ===================== loader =====================
    if (lane == 0) {
      const uint32_t box_bytes = (uint32_t)((p.TW + (copies == 1 ? 2 : 0)) * (p.R + 2) * 128);
      int u = 0;
      for (int tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
        const int a = fast_div(tile, inv_pa), rem = tile - a * per_a;
        const int kb = fast_div(rem, inv_lb), lb = rem - kb * p.LB;
        const int k0 = kb * p.R, l0 = lb * p.TW;
        for (int c = 0; c < copies; ++c, ++u) {
          const int s = u % ring;
          mbar_wait(&empty_bar[s], ((uint32_t)(u / ring) & 1u) ^ 1u);
          mbar_expect_tx(&full_bar[s], box_bytes);
          tma_load_4d(&hmap, &full_bar[s], smem + (size_t)s * p.unit_bytes, 0, l0 - 1 + c, k0 - 1, a);
        }
      }
    }
  } else if (wgi >= 1) {
    // ===================== MMA + epilogue: warpgroup wg owns MMA rows 64 wg .. 64 wg + 63 =====================
    const int wg = wgi - 1, wl = warp & 3;
    const bool leader = threadIdx.x % 128 == 0;
    const int t = lane & 3;
    const int m0 = wg * 64 + 16 * wl + (lane >> 2);          // fragment rows m0 and m0 + 8
    float sx, sh;
    nc_scales(p, sx, sh);
    const float inv = p.inv_sw2 / sh;
    const uint32_t wbase = smem_u32(wsm), sbase = smem_u32(smem);
    const uint32_t tk_stride = (uint32_t)(p.P * 128);
    int u = 0;
    for (int tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
      float da[2][16], db[2][8];       // per net: [0,8) hi*hi, [8,16) hi*lo fragments ; lo*hi
#pragma unroll
      for (int c = 0; c < COPIES; ++c, ++u) {
        const int s = u % ring;
        mbar_wait(&full_bar[s], (uint32_t)(u / ring) & 1u);
        const uint32_t blk = sbase + (uint32_t)(s * p.unit_bytes) + (uint32_t)(wg * 64 * 128);
        wgmma_fence();
#pragma unroll
        for (int j = 0; j < (COPIES == 1 ? 3 : 1); ++j) {        // taps in (tl outer, tk inner) order for either layout
          const int tlx = COPIES == 1 ? j : c;
#pragma unroll
          for (int tk = 0; tk < 3; ++tk) {
            // 128-byte granular start, base offset 0 (see above)
            const uint64_t adesc = make_sw128_desc(blk + (uint32_t)tk * tk_stride + (COPIES == 1 ? (uint32_t)(tlx * 128) : 0u));
            const uint64_t wdesc = make_sw128_desc(wbase + (uint32_t)((tk * 3 + tlx) * kL2WTap));
            const uint32_t acc = (tlx > 0 || tk > 0) ? 1u : 0u;
#pragma unroll
            for (int net = 0; net < 2; ++net) {
              wgmma_f16<32>(da[net], adesc + 2 * (net * 2), wdesc + 2 * net, acc);       // hi*hi | hi*lo
              wgmma_f16<16>(db[net], adesc + 2 * (net * 2 + 1), wdesc + 2 * net, acc);   // lo*hi
            }
          }
        }
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_regs<16>(da[0]);
        wgmma_fence_regs<16>(da[1]);
        wgmma_fence_regs<8>(db[0]);
        wgmma_fence_regs<8>(db[1]);
        mbar_arrive_if(&empty_bar[s], leader);
      }
      const int a = fast_div(tile, inv_pa), rem = tile - a * per_a;
      const int kb = fast_div(rem, inv_lb), lb = rem - kb * p.LB;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int m = m0 + 8 * h;
        const int kk = m / p.P, ll = m - kk * p.P;
        const int k = kb * p.R + kk, l = lb * p.TW + ll;
        if (kk < p.R && ll < p.TW && k < p.hB && l < p.wB) {
          const size_t v = (size_t)a * p.nB + (size_t)k * p.wB + l;
#pragma unroll
          for (int net = 0; net < 2; ++net)
#pragma unroll
            for (int j = 0; j < 2; ++j)
#pragma unroll
              for (int e = 0; e < 2; ++e) {
                const int d = 8 * j + 2 * t + e, i = 4 * j + 2 * h + e;
                if (d < 9) p.partial[(size_t)(net * 9 + d) * p.V + v] = ((db[net][i] + da[net][8 + i]) + da[net][i]) * inv;
              }
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// max |x| (device-side activation scale of the tensor-core NC path)
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) absmax_kernel(const float* __restrict__ x, size_t n, unsigned int* __restrict__ out) {
  float m = 0.f;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    m = fmaxf(m, fabsf(x[i]));
  m = warp_max(m);
  if ((threadIdx.x & 31) == 0) atomicMax(out, __float_as_uint(m));   // non-negative floats order like their bits
}

int launch_absmax(const float* x, size_t n, unsigned int* out, cudaStream_t st) {
  P2P_CUDA_OK(cudaMemsetAsync(out, 0, sizeof(unsigned int), st));
  const int blocks = (int)((n + 255) / 256 < 1184 ? (n + 255) / 256 : 1184);
  absmax_kernel<<<blocks, 256, 0, st>>>(x, n, out);
  P2P_LAUNCH_OK();
  return 0;
}

// ------------------------------------------------------------------------------------------------
// combine: out[a][b] = sum_net relu(b2 + sum_(ta,tb) P[net][ta*3+tb][a + (ta-1, tb-1)][b]), fused with the
// row / column maxima of the MutualMatching that follows (rowmax[a] = max_b, colmax[b] = max_a).
// Block = kCombineRows A cells; the 9 neighbour offsets are block-uniform.
// ------------------------------------------------------------------------------------------------
constexpr int kCombineRows = 2;      // A cells per block: nA / 2 blocks keep every SM busy with several blocks

// VEC = 4: float4 columns (nB % 4 == 0).  Every neighbour plane is loaded unconditionally from a clamped (always valid)
// cell and masked afterwards, so the 18 loads of an output element are independent and in flight together.
template <int VEC>
__global__ void __launch_bounds__(1024) nc_combine_kernel(const float* __restrict__ P, int hA, int wA, int nB, float b2,
                                                        float* __restrict__ out, float* __restrict__ rowmax,
                                                        unsigned int* __restrict__ colmax) {
  constexpr int R = kCombineRows;
  __shared__ float red[32][R];
  const int nA = hA * wA;
  const size_t V = (size_t)nA * nB;
  const int r0 = blockIdx.x * R;
  float rm[R];
#pragma unroll
  for (int r = 0; r < R; ++r) rm[r] = -INFINITY;
  for (int col = threadIdx.x * VEC; col < nB; col += (int)blockDim.x * VEC) {
    float cm[VEC];
#pragma unroll
    for (int e = 0; e < VEC; ++e) cm[e] = -INFINITY;
#pragma unroll
    for (int r = 0; r < R; ++r) {
      const int a = r0 + r;
      if (a >= nA) continue;
      const int ia = a / wA, ja = a - ia * wA;
      float v[2][9][VEC];
      bool ok[9];
#pragma unroll
      for (int d = 0; d < 9; ++d) {
        const int i2 = ia + d / 3 - 1, j2 = ja + d % 3 - 1;
        ok[d] = i2 >= 0 && i2 < hA && j2 >= 0 && j2 < wA;
        const size_t cell = ok[d] ? (size_t)(i2 * wA + j2) : (size_t)a;
#pragma unroll
        for (int net = 0; net < 2; ++net) {
          const float* src = P + (size_t)(net * 9 + d) * V + cell * nB + col;
          if (VEC == 4) {
            const float4 q = __ldg(reinterpret_cast<const float4*>(src));
            v[net][d][0] = q.x; v[net][d][VEC > 1 ? 1 : 0] = q.y; v[net][d][VEC > 2 ? 2 : 0] = q.z; v[net][d][VEC > 3 ? 3 : 0] = q.w;
          } else {
            v[net][d][0] = __ldg(src);
          }
        }
      }
      float tot[VEC];
#pragma unroll
      for (int e = 0; e < VEC; ++e) {
        tot[e] = 0.f;
#pragma unroll
        for (int net = 0; net < 2; ++net) {
          float acc = b2;
#pragma unroll
          for (int d = 0; d < 9; ++d) acc += ok[d] ? v[net][d][e] : 0.f;     // same order as before; adding +0 is exact
          tot[e] += fmaxf(acc, 0.f);
        }
        rm[r] = fmaxf(rm[r], tot[e]);
        cm[e] = fmaxf(cm[e], tot[e]);
      }
      float* o = out + (size_t)a * nB + col;
      if (VEC == 4) *reinterpret_cast<float4*>(o) = make_float4(tot[0], tot[VEC > 1 ? 1 : 0], tot[VEC > 2 ? 2 : 0], tot[VEC > 3 ? 3 : 0]);
      else o[0] = tot[0];
    }
    if (colmax != nullptr) {
#pragma unroll
      for (int e = 0; e < VEC; ++e) atomicMax(colmax + col + e, f2ord(cm[e]));
    }
  }
  if (rowmax == nullptr) return;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
  for (int r = 0; r < R; ++r) {
    const float v = warp_max(rm[r]);
    if (lane == 0) red[wid][r] = v;
  }
  __syncthreads();
  if (threadIdx.x < R && r0 + threadIdx.x < nA) {
    float v = red[0][threadIdx.x];
    for (int wv = 1; wv < (int)(blockDim.x >> 5); ++wv) v = fmaxf(v, red[wv][threadIdx.x]);
    rowmax[r0 + threadIdx.x] = v;
  }
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
static float pow2_scale_for(float maxabs, float target_hi) {   // power of two s: maxabs * s in [target_hi/2, target_hi)
  if (!(maxabs > 0.f) || !isfinite(maxabs)) return 1.f;
  int e, et;
  frexpf(maxabs, &e);
  frexpf(target_hi, &et);
  return ldexpf(1.f, et - 1 - e);
}

// element (n, k) of a [rows][64] K-major 128B-swizzled atom
static inline size_t sw128_index(int n, int k) { return (size_t)n * 64 + ((((k >> 3) ^ (n & 7)) << 3) | (k & 7)); }

int nc_umma_pack(const float* w1p, const float* b1p, const float* w2p, NcUmmaWeights& W) {
  float m1 = 0.f, m2 = 0.f, wsum = 0.f, b1max = 0.f;
  for (int i = 0; i < 81 * 32; ++i) {
    m1 = fmaxf(m1, fabsf(w1p[i]));
    m2 = fmaxf(m2, fabsf(w2p[i]));
  }
  for (int c = 0; c < 32; ++c) {
    float s = 0.f;
    for (int t = 0; t < 81; ++t) s += fabsf(w1p[t * 32 + c]);
    wsum = fmaxf(wsum, s);
    b1max = fmaxf(b1max, fabsf(b1p[c]));
  }
  const float s1 = pow2_scale_for(m1, 1024.f), s2 = pow2_scale_for(m2, 1024.f);
  W.wsum1 = wsum * 1.0001f;
  W.b1max = b1max;
  W.inv_sw1 = 1.f / s1;
  W.inv_sw2 = 1.f / s2;
  // layer 1: [atom 0..1][hi 32 rows | lo 32 rows][64]; k = tap (81 used)
  std::vector<__half> img1((size_t)2 * 64 * 64, __float2half(0.f));
  for (int c = 0; c < 32; ++c)
    for (int t = 0; t < 81; ++t) {
      const float v = w1p[t * 32 + c] * s1;
      const __half h = __float2half_rn(v), l = __float2half_rn(v - __half2float(h));
      const int atom = t >> 6, k = t & 63;
      img1[(size_t)atom * 64 * 64 + sw128_index(c, k)] = h;
      img1[(size_t)atom * 64 * 64 + sw128_index(32 + c, k)] = l;
    }
  // layer 2: [B tap 0..8][32 rows][64]; rows 0..15 = hi, 16..31 = lo parts of partial map (ta,tb) (9 used each),
  // k = net * 16 + channel (K16 slice = net)
  std::vector<__half> img2((size_t)9 * 32 * 64, __float2half(0.f));
  for (int net = 0; net < 2; ++net)
    for (int d = 0; d < 9; ++d)
      for (int t = 0; t < 9; ++t)
        for (int ch = 0; ch < 16; ++ch) {
          const float v = w2p[(d * 9 + t) * 32 + net * 16 + ch] * s2;
          const __half h = __float2half_rn(v), l = __float2half_rn(v - __half2float(h));
          img2[(size_t)t * 32 * 64 + sw128_index(d, net * 16 + ch)] = h;
          img2[(size_t)t * 32 * 64 + sw128_index(16 + d, net * 16 + ch)] = l;
        }
  const size_t b1 = img1.size() * 2, b2 = img2.size() * 2;
  if (W.blob == nullptr) {
    if (cudaMalloc(&W.blob, b1 + b2) != cudaSuccess) {
      cudaGetLastError();
      set_last_error("out of device memory packing the NC weights");
      return -3;
    }
  }
  W.img1 = reinterpret_cast<__half*>(W.blob);
  W.img2 = reinterpret_cast<__half*>(W.blob + b1);
  P2P_CUDA_OK(cudaMemcpy(W.img1, img1.data(), b1, cudaMemcpyHostToDevice));
  P2P_CUDA_OK(cudaMemcpy(W.img2, img2.data(), b2, cudaMemcpyHostToDevice));
  return 0;
}

size_t nc_umma_scratch_bytes(size_t V) { return V * 128 + 18 * V * 4 + 4096; }

constexpr int kL1SmemBudget = 225 * 1024;
constexpr int kL1SmemFixed = kL1Stages * 2 * kNcAtom + 2 * 64 * 128 + 2 * kNcAtom + 1024;   // operand ring, weights, store staging

// Padded row pitch of xp (words) and the number of layer-1 staging buffers.  Preferred pitch: a multiple of 4 words
// (16-byte bulk copies) that is == wB + 32..35, so that the lanes of a warp -- consecutive B cells, which wrap to the
// next row mid-warp -- still hit 32 distinct shared-memory banks; very narrow or very wide grids fall back to the
// compact pitch wB + 2..5 and / or a single buffer when the staging block would not fit.
static void nc_l1_staging(int wB, int& pitch, int& bufs) {
  const int wide = (wB + 32 + 3) & ~3, compact = (wB + 2 + 3) & ~3;
  const int cand[4][2] = {{wide, 2}, {compact, 2}, {wide, 1}, {compact, 1}};
  for (int i = 0; i < 4; ++i) {
    pitch = cand[i][0];
    bufs = cand[i][1];
    if (kL1SmemFixed + bufs * 9 * nc_l1_rows(wB) * pitch * 4 <= kL1SmemBudget) return;
  }
}
static int nc_pitch(int wB) {
  int pitch, bufs;
  nc_l1_staging(wB, pitch, bufs);
  return pitch;
}
size_t nc_umma_xp_bytes(int hA, int wA, int hB, int wB) {
  return ((size_t)(hA + 2) * (wA + 2) * (hB + 2) + nc_l1_rows(wB)) * nc_pitch(wB) * 4 + 256;
}

// Layer-2 tiling: the (TW, R) with the fewest tiles; mode 0 compares both block layouts (ties: one haloed block).
static void nc_l2_geometry(int hB, int wB, int mode, int ctas, NcParams& p) {
  long long best = -1;
  for (int copies = 1; copies <= 3; copies += 2) {
    if ((mode == 1 && copies != 1) || (mode == 2 && copies != 3)) continue;
    for (int tw = wB < 128 ? wB : 128; tw >= 1; --tw) {
      const int P = tw + (copies == 1 ? 2 : 0);
      if (P > 128 && copies == 1 && tw > 126) continue;
      const int R = (128 - tw) / P + 1;
      const long long n = (long long)cdiv(wB, tw) * cdiv(hB, R);
      if (best < 0 || n < best) {
        best = n;
        p.copies = copies; p.TW = tw; p.R = R; p.P = P;
      }
    }
  }
  p.KB = cdiv(hB, p.R);
  p.LB = cdiv(wB, p.TW);
  const int lines_box = (p.R + 2) * p.P, lines_read = 128 + 2 * p.P + 2;
  p.unit_bytes = (int)align_up((size_t)(lines_box > lines_read ? lines_box : lines_read) * 128, 1024);
  p.l2_ctas = ctas;
  p.ring = (int)(((ctas == 2 ? 110 : 200) * 1024 - 9 * kL2WTap) / p.unit_bytes);
  if (p.ring < 1 && ctas == 2) {
    p.l2_ctas = 1;
    p.ring = (int)((200 * 1024 - 9 * kL2WTap) / p.unit_bytes);
  }
  if (p.ring > kL2MaxRing) p.ring = kL2MaxRing;
}

// x [hA*wA][hB*wB] -> out (NeighConsensus output); rowmax / colmax (optional) receive the maxima MutualMatching needs.
// xmax: device word holding the float bits of max |x| (launch_absmax or the fused mutual_apply pass).
// xp: scratch of nc_umma_xp_bytes().  l2_mode: 0 auto, 1 one haloed block per tile, 2 one block per column tap; + 8: one
// layer-2 CTA per SM instead of two.
int launch_neigh_consensus_umma(const float* x, int hA, int wA, int hB, int wB, const NcUmmaWeights& W, const float* b1p,
                                float b2, const unsigned int* xmax, uint32_t* xp, __half* hidden, float* partial,
                                float* out, float* rowmax, unsigned int* colmax, int l2_mode, int num_sms, cudaStream_t st) {
  NcParams p;
  memset(&p, 0, sizeof(p));
  p.hA = hA; p.wA = wA; p.hB = hB; p.wB = wB;
  p.nA = hA * wA; p.nB = hB * wB;
  p.V = (long long)p.nA * p.nB;
  p.x = x; p.xmax = xmax; p.xp = xp; p.hidden = hidden; p.partial = partial; p.b1p = b1p;
  p.wsum1 = W.wsum1; p.b1max = W.b1max; p.inv_sw1 = W.inv_sw1; p.inv_sw2 = W.inv_sw2;
  p.WP = nc_pitch(wB);
  const long long t1 = (long long)p.nA * ((p.nB + 127) / 128);
  P2P_REQUIRE(t1 < (1ll << 22) && p.nB < (1 << 22), "NeighConsensus: 4D volume too large");
  nc_pad_split_kernel<<<(hA + 2) * (wA + 2), 256, 0, st>>>(p);
  P2P_LAUNCH_OK();
  {
    p.wimg = W.img1;
    p.tiles = (int)t1;
    int pitch;
    nc_l1_staging(wB, pitch, p.l1_bufs);
    const int smem = kL1SmemFixed + p.l1_bufs * 9 * nc_l1_rows(wB) * p.WP * 4;
    P2P_REQUIRE(pitch == p.WP && smem <= kL1SmemBudget,
                "NeighConsensus layer 1: B grid too wide for the shared-memory staging (wB <= ~340)");
    CUtensorMap hstore;
    const uint64_t dims[3] = {64, (uint64_t)p.nB, (uint64_t)p.nA};
    const uint64_t strides[2] = {128, (uint64_t)p.nB * 128};
    const uint32_t box[3] = {64, 128, 1};
    int rc = make_tmap_fp16(&hstore, hidden, 3, dims, strides, box);
    if (rc) return rc;
    auto k = nc_l1_umma_kernel;
    P2P_ENSURE_SMEM(k, smem);
    const int grid = p.tiles < num_sms ? p.tiles : num_sms;
    k<<<grid, kL1Threads, smem, st>>>(p, hstore);
    P2P_LAUNCH_OK();
  }
  {
    p.wimg = W.img2;
    nc_l2_geometry(hB, wB, l2_mode & 3, (l2_mode & 8) ? 1 : 2, p);      // +8 (development): one CTA per SM
    const long long t2 = (long long)p.nA * p.KB * p.LB;
    P2P_REQUIRE(t2 < (1ll << 22), "NeighConsensus: 4D volume too large");
    P2P_REQUIRE(p.ring >= 1, "NeighConsensus layer 2: block buffer does not fit in shared memory");
    p.tiles = (int)t2;
    CUtensorMap hmap;
    const uint64_t dims[4] = {64, (uint64_t)wB, (uint64_t)hB, (uint64_t)p.nA};
    const uint64_t strides[3] = {128, (uint64_t)wB * 128, (uint64_t)p.nB * 128};
    const uint32_t box[4] = {64, (uint32_t)(p.TW + (p.copies == 1 ? 2 : 0)), (uint32_t)(p.R + 2), 1};
    int rc = make_tmap_fp16(&hmap, hidden, 4, dims, strides, box);
    if (rc) return rc;
    const int smem = p.ring * p.unit_bytes + 9 * kL2WTap + 1024;
    const int slots = num_sms * p.l2_ctas;
    const int grid = p.tiles < slots ? p.tiles : slots;
#define P2P_NC_L2_LAUNCH(C, T)                    \
  {                                               \
    auto k = nc_l2_umma_kernel<C, T>;             \
    P2P_ENSURE_SMEM(k, smem);                     \
    k<<<grid, 384, smem, st>>>(p, hmap);          \
  }
    if (p.copies == 1 && p.l2_ctas == 1) P2P_NC_L2_LAUNCH(1, 1)
    else if (p.copies == 1) P2P_NC_L2_LAUNCH(1, 2)
    else if (p.l2_ctas == 1) P2P_NC_L2_LAUNCH(3, 1)
    else P2P_NC_L2_LAUNCH(3, 2)
#undef P2P_NC_L2_LAUNCH
    P2P_LAUNCH_OK();
  }
  if (colmax != nullptr) P2P_CUDA_OK(cudaMemsetAsync(colmax, 0, sizeof(unsigned int) * p.nB, st));
  // block = one pass over the columns of its rows when they fit (nB = 1200 -> 300 float4 columns -> 320 threads)
  const int vec = p.nB % 4 == 0 ? 4 : 1;
  int threads = (cdiv(p.nB, vec) + 31) & ~31;
  threads = threads > 1024 ? 1024 : (threads < 64 ? 64 : threads);
  if (vec == 4)
    nc_combine_kernel<4><<<cdiv(p.nA, kCombineRows), threads, 0, st>>>(partial, hA, wA, p.nB, b2, out, rowmax, colmax);
  else
    nc_combine_kernel<1><<<cdiv(p.nA, kCombineRows), threads, 0, st>>>(partial, hA, wA, p.nB, b2, out, rowmax, colmax);
  P2P_LAUNCH_OK();
  return 0;
}

}  // namespace p2p
