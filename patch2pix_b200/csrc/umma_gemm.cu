// wgmma implicit-GEMM kernel for sm_90a: TMA-staged fp16 operand tiles in shared memory (128B swizzle,
// K-major), wgmma.mma_async (f16 inputs, fp32 accumulate in registers), shared-memory-staged epilogue.
//
// One kernel serves four contractions of the Patch2Pix hot path (reference file:line):
//   conv1 of FeatRegressNet  (Conv2d 518->512 k3 s2 p1 + BN)       networks/modules.py:76-87,103-105
//   conv2 of FeatRegressNet  (Conv2d 512->512 k3 s1 p1 + BN, ReLU, MaxPool 8)   same
//   the two big Linear layers of the regressor head (+ BN1d, ReLU)
//   FeatCorrelation + maxpool4d (C x n1 x n2 contraction + 2^4 max)  networks/modules.py:11-53
//
// Precision: operands are fp16 "hi" (+ optional fp16 "lo" residual) pairs of scaled fp32 values.
//   PASSES = 1:  hi*hi                      (fp16-grade inputs, fp32 accumulate)
//   PASSES = 3:  lo*hi + hi*lo + hi*hi      (~2^-22 relative products, i.e. fp32-grade)
// SEGMENTED accumulation: the tensor core accumulates only `seg_len` k-steps at a time; each partial sum is
// added to fp32 register totals with round-to-nearest, which bounds the accumulator-rounding drift of long K chains.
#include <cuda.h>

#include <vector>

#include "kernels.h"
#include "umma_gemm.h"
#include "umma_ptx.cuh"

namespace p2p {

// ------------------------------------------------------------------------------------------------
// epilogues: consume one piece of 32 accumulator columns of one row
// ------------------------------------------------------------------------------------------------
// WindowShare partial sums of one staged piece (32 fp32 accumulators of one tile row, `srow` in shared memory): a prefix
// launch stores them, a continuation adds its half-group's prefix to them in place, in shared memory: the consumers
// hold the tile's other accumulators meanwhile, and a register copy of the piece beside the prefix would spill.
// split_slot = first class-1 slot.
// Partial-sum layout [unit][256-column half][64 rows][256]: what one 128 x 256 tile reads of one slot is one
// contiguous 64 KB block, which the producer prefetches into L2 while the tile's main loop runs.
__device__ __forceinline__ size_t part_offset(int unit, int row64, int col) {
  return (((size_t)unit * 2 + (col >> 8)) * 64 + row64) * 256 + (col & 255);
}
__device__ __forceinline__ int part_unit(int slot, int split_slot, int split_unit) {
  return slot < split_slot ? slot >> 2 : split_unit + ((slot - split_slot) >> 2);
}
__device__ __forceinline__ void share_piece(const WindowShare& ws, int split_slot, int split_unit, int n_patches, int m_tile,
                                            int row, int col0, float* srow) {
  const int n = m_tile * 2 + (row >> 6);
  if (n >= n_patches) return;
  if (ws.part_out != nullptr) {
    float4* dst = reinterpret_cast<float4*>(ws.part_out + part_offset(n, row & 63, col0));
#pragma unroll 1
    for (int q = 0; q < 8; ++q) dst[q] = make_float4(srow[4 * q], srow[4 * q + 1], srow[4 * q + 2], srow[4 * q + 3]);
  } else {
    const float4* src = reinterpret_cast<const float4*>(ws.part_in + part_offset(part_unit(n, split_slot, split_unit), row & 63, col0));
    float4 a8[8];                       // all 8 loads in flight at once (this piece's accumulators are staged already)
#pragma unroll
    for (int q = 0; q < 8; ++q) a8[q] = __ldg(src + q);
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      const float4 a = a8[q];
      srow[4 * q] += a.x;
      srow[4 * q + 1] += a.y;
      srow[4 * q + 2] += a.z;
      srow[4 * q + 3] += a.w;
    }
  }
}

// SHARE (AMODE_WINDOW): the conv1 outputs go to row ws.slot_row[slot]
template <int EPI, bool SHARE>
__device__ __forceinline__ void epilogue_piece(const UmmaEpilogue& e, const WindowShare& ws, int n_patches, int m_tile,
                                               int row, int col0, const float* v) {
  if (EPI == EPI_PLAIN) {
    const int r = m_tile * 128 + row;
    if (r < e.m_rows) {
      float* dst = e.c + (size_t)r * e.ldc + col0;
#pragma unroll
      for (int i = 0; i < 32; ++i)
        if (col0 + i < e.n_cols) dst[i] = v[i] * e.alpha;
    }
  } else if (EPI == EPI_CONV1) {
    const int n = m_tile * 2 + (row >> 6);
    if (n < n_patches) {
      const int r = SHARE && ws.slot_row != nullptr ? __ldg(ws.slot_row + n) : n;   // the conv1 output row
      __align__(16) __half h[32];
      __align__(16) __half l[32];
#pragma unroll
      for (int i = 0; i < 32; ++i) {
        const float y = fmaf(v[i], __ldg(e.scale + col0 + i), __ldg(e.bias + col0 + i)) * e.y_scale;
        h[i] = __float2half_rn(y);
        l[i] = __float2half_rn(y - __half2float(h[i]));
      }
      const size_t o = ((size_t)r * 64 + (row & 63)) * 512 + col0;
#pragma unroll
      for (int q = 0; q < 4; ++q) reinterpret_cast<uint4*>(e.y_hi + o)[q] = reinterpret_cast<const uint4*>(h)[q];
      if (e.y_lo != nullptr) {
#pragma unroll
        for (int q = 0; q < 4; ++q) reinterpret_cast<uint4*>(e.y_lo + o)[q] = reinterpret_cast<const uint4*>(l)[q];
      }
      // zero this patch's slice of the max-pool accumulator that conv2's epilogue merges into with atomicMax
      // (replaces a cudaMemsetAsync between the two convolutions)
      if (e.pooled != nullptr && (row & 63) == 0) {
        float4* z = reinterpret_cast<float4*>(e.pooled + (size_t)r * 512 + col0);
#pragma unroll
        for (int q = 0; q < 8; ++q) z[q] = make_float4(0.f, 0.f, 0.f, 0.f);
      }
    }
  } else if (EPI == EPI_CONV2) {
    // relu + max over the 32 rows held by this warp (half a patch); atomically merged in HBM
    const int n = m_tile * 2 + (row >> 6);
    const int lane = threadIdx.x & 31;
    unsigned int mine = 0;
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      const float y = fmaxf(fmaf(v[i], __ldg(e.scale + col0 + i), __ldg(e.bias + col0 + i)), 0.f);
      const unsigned int m = __reduce_max_sync(0xffffffffu, __float_as_uint(y));
      if (lane == i) mine = m;
    }
    if (n < n_patches) atomicMax(reinterpret_cast<unsigned int*>(e.pooled) + (size_t)n * 512 + col0 + lane, mine);
  } else if (EPI == EPI_FC) {
    // Linear + folded BatchNorm1d + ReLU; output re-split to fp16 hi/lo as the next layer's A operand
    const int r = m_tile * 128 + row;
    if (r < n_patches) {
      __align__(16) __half h[32];
      __align__(16) __half l[32];
#pragma unroll
      for (int i = 0; i < 32; ++i) {
        // saturate instead of overflowing to inf (an activation beyond 65504 / y_scale is outside the fp16 operand range)
        const float y = fminf(fmaxf(fmaf(v[i], __ldg(e.scale + col0 + i), __ldg(e.bias + col0 + i)), 0.f) * e.y_scale, 65504.f);
        h[i] = __float2half_rn(y);
        l[i] = __float2half_rn(y - __half2float(h[i]));
      }
      const size_t o = (size_t)r * e.ldc + col0;
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        reinterpret_cast<uint4*>(e.y_hi + o)[q] = reinterpret_cast<const uint4*>(h)[q];
        reinterpret_cast<uint4*>(e.y_lo + o)[q] = reinterpret_cast<const uint4*>(l)[q];
      }
    }
  } else if (EPI == EPI_CORR) {
    // rows/cols are in pooling-window order: 4 rows x 4 cols = one 4D window
    const int lane = threadIdx.x & 31;
    const int pa = m_tile * 128 + row;
    const int ca = pa >> 2, mi = pa & 3;
#pragma unroll
    for (int cell = 0; cell < 8; ++cell) {
      float best = v[cell * 4];
      int code = mi * 4;
#pragma unroll
      for (int j = 1; j < 4; ++j)
        if (v[cell * 4 + j] > best) {
          best = v[cell * 4 + j];
          code = mi * 4 + j;
        }
#pragma unroll
      for (int o = 1; o <= 2; o <<= 1) {
        const float b2 = __shfl_xor_sync(0xffffffffu, best, o);
        const int c2 = __shfl_xor_sync(0xffffffffu, code, o);
        if (b2 > best || (b2 == best && c2 < code)) {
          best = b2;
          code = c2;
        }
      }
      const int cb = (col0 >> 2) + cell;
      if ((lane & 3) == 0 && ca < e.np1 && cb < e.np2) {
        e.c[(size_t)ca * e.np2 + cb] = best * e.alpha;
        e.code[(size_t)ca * e.np2 + cb] = (uint8_t)code;
      }
    }
  }
}

__device__ __forceinline__ void named_bar(int id, int threads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory");
}

// ------------------------------------------------------------------------------------------------
// fragment epilogues of the 256-wide 1-pass conv launches: straight from the wgmma accumulators
// ------------------------------------------------------------------------------------------------
// Consumer warpgroup wg owns patch n = 2 m_tile + wg (its 64 rows).  Thread 32 wl + lane holds rows fr = 16 wl + lane / 4
// and fr + 8, columns 8 j + fc, +1 (fc = 2 (lane % 4), j = 0..31) as acc[4 j + {0, 1, 2, 3}] (umma_ptx.cuh).  The
// per-element arithmetic and the pooling max are epilogue_piece's, so both epilogues write identical bits; these skip
// the fp32 staging round trip, its 8 named barriers per tile and the per-element scale / bias loads.
constexpr int kFragBox = 64 * 128;   // one 128B-swizzled TMA box: 64 rows x 64 fp16

// one step of a max reduce-scatter across lanes l and l ^ (H / 2): the lane with that bit set keeps the upper half
template <int H>
__device__ __forceinline__ void reduce_scatter_half(uint32_t* m, int lane) {
  const bool up = (lane & (H / 2)) != 0;
#pragma unroll
  for (int i = 0; i < H; ++i) {
    const uint32_t give = up ? m[i] : m[i + H], keep = up ? m[i + H] : m[i];
    m[i] = max(keep, __shfl_xor_sync(0xffffffffu, give, H / 2));
  }
}

// conv2: relu(BN), max over the patch's 64 rows, one atomicMax per column.  red: this warpgroup's [4 warps][256];
// sb: the CTA's copy of scale[512] then bias[512] in shared memory.
__device__ __forceinline__ void conv2_frag(const UmmaEpilogue& e, const float* acc, int n, int n_units, int col0,
                                           uint32_t* red, const float* sb, int wg) {
  const int lane = threadIdx.x & 31, wl = (threadIdx.x >> 5) & 3, fc = 2 * (lane & 3);
  uint32_t m[64];   // m[2 j + b]: max over the thread's two rows of column 8 j + fc + b (as uint, like the atomicMax)
#pragma unroll
  for (int j = 0; j < 32; ++j) {
    const float2 s = *reinterpret_cast<const float2*>(sb + col0 + 8 * j + fc);
    const float2 b = *reinterpret_cast<const float2*>(sb + 512 + col0 + 8 * j + fc);
    m[2 * j] = max(__float_as_uint(fmaxf(fmaf(acc[4 * j], s.x, b.x), 0.f)),
                   __float_as_uint(fmaxf(fmaf(acc[4 * j + 2], s.x, b.x), 0.f)));
    m[2 * j + 1] = max(__float_as_uint(fmaxf(fmaf(acc[4 * j + 1], s.y, b.y), 0.f)),
                       __float_as_uint(fmaxf(fmaf(acc[4 * j + 3], s.y, b.y), 0.f)));
  }
  // reduce-scatter over the warp's 8 row pairs (lane bits 4, 3, 2): 32 + 16 + 8 shuffles, after which m[i], i < 8, is
  // the warp's max of index 8 (lane / 4) + i, i.e. column 32 (lane / 4) + 8 (i / 2) + fc + i % 2
  reduce_scatter_half<32>(m, lane);
  reduce_scatter_half<16>(m, lane);
  reduce_scatter_half<8>(m, lane);
  named_bar(1 + wg, 128);   // the previous tile's reads of red are done
#pragma unroll
  for (int i = 0; i < 8; i += 2)
    *reinterpret_cast<uint2*>(red + wl * 256 + 32 * (lane >> 2) + 4 * i + fc) = make_uint2(m[i], m[i + 1]);
  named_bar(1 + wg, 128);
  if (n < n_units) {
    const int t = threadIdx.x & 127;
    uint2 v = *reinterpret_cast<const uint2*>(red + 2 * t);
#pragma unroll
    for (int w = 1; w < 4; ++w) {
      const uint2 u = *reinterpret_cast<const uint2*>(red + w * 256 + 2 * t);
      v.x = max(v.x, u.x);
      v.y = max(v.y, u.y);
    }
    unsigned int* dst = reinterpret_cast<unsigned int*>(e.pooled) + (size_t)n * 512 + col0 + 2 * t;
    atomicMax(dst, v.x);
    atomicMax(dst + 1, v.y);
  }
}

// conv1: BN (* y_scale) to fp16 in the fragment layout, stmatrix into 128B-swizzled boxes, TMA store at the patch's
// output row; the two 128-column halves go one after the other through one 16 KB buffer (buf) per warpgroup, whose
// reuse waits until the previous store has read it.  A prefix launch (SHARE, part_out) stores its raw fp32 sums
// instead, fragment-direct (8 lanes x 32 contiguous bytes per row); a continuation adds its prefix sums first.
template <bool SHARE>
__device__ __forceinline__ void conv1_frag(const UmmaGemmParams& p, float* acc, int n, int n_units, int split_slot,
                                           int split_unit, int col0, uint8_t* buf) {
  if (n >= n_units) return;   // warpgroup-uniform: the pad patch of an odd count
  const int lane = threadIdx.x & 31, wl = (threadIdx.x >> 5) & 3, fc = 2 * (lane & 3), fr = 16 * wl + (lane >> 2);
  const int wg = threadIdx.x / 128 - 1, t = threadIdx.x & 127;
  const WindowShare& ws = p.ws;
  if (SHARE && ws.part_out != nullptr) {   // prefix launch: no BN, no y_hi, no pooled zeroing
    float* dst = ws.part_out + part_offset(n, 0, col0);
#pragma unroll
    for (int j = 0; j < 32; ++j)
#pragma unroll
      for (int h = 0; h < 2; ++h)
        *reinterpret_cast<float2*>(dst + (fr + 8 * h) * 256 + 8 * j + fc) = make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
    return;
  }
  if (SHARE && ws.part_in != nullptr) {
    const float* src = ws.part_in + part_offset(part_unit(n, split_slot, split_unit), 0, col0);
#pragma unroll
    for (int j0 = 0; j0 < 32; j0 += 8) {
      float2 a[16];                     // 16 loads in flight at a time
#pragma unroll
      for (int i = 0; i < 16; ++i)
        a[i] = __ldg(reinterpret_cast<const float2*>(src + (fr + 8 * (i & 1)) * 256 + 8 * (j0 + (i >> 1)) + fc));
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        acc[4 * (j0 + (i >> 1)) + 2 * (i & 1)] += a[i].x;
        acc[4 * (j0 + (i >> 1)) + 2 * (i & 1) + 1] += a[i].y;
      }
    }
  }
  const int r = SHARE && ws.slot_row != nullptr ? __ldg(ws.slot_row + n) : n;   // the conv1 output row
  // zero this patch's slice of the max-pool accumulator that conv2's epilogue merges into with atomicMax
  if (p.epi.pooled != nullptr)
    *reinterpret_cast<float2*>(p.epi.pooled + (size_t)r * 512 + col0 + 2 * t) = make_float2(0.f, 0.f);
  const float ys = p.epi.y_scale;
  const uint32_t sbuf = smem_u32(buf);
  const int mi = lane >> 3, rr = lane & 7;           // this lane's stmatrix address: row rr of matrix mi
  const uint32_t arow = sbuf + (uint32_t)(16 * wl + 8 * (mi & 1) + rr) * 128;
#pragma unroll
  for (int hf = 0; hf < 2; ++hf) {
    if (t == 0) bulk_wait_group_read<0>();   // the previous store out of buf has read it
    named_bar(1 + wg, 128);
#pragma unroll
    for (int j = 16 * hf; j < 16 * hf + 16; j += 2) {
      uint32_t hv[4];                          // matrices (j, rows fr), (j, fr + 8), (j + 1, fr), (j + 1, fr + 8)
#pragma unroll
      for (int q = 0; q < 2; ++q) {
        const float2 s = __ldg(reinterpret_cast<const float2*>(p.epi.scale + col0 + 8 * (j + q) + fc));
        const float2 b = __ldg(reinterpret_cast<const float2*>(p.epi.bias + col0 + 8 * (j + q) + fc));
        const float* d = acc + 4 * (j + q);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const __half2 y = __floats2half2_rn(fmaf(d[2 * h], s.x, b.x) * ys, fmaf(d[2 * h + 1], s.y, b.y) * ys);
          hv[2 * q + h] = *reinterpret_cast<const uint32_t*>(&y);
        }
      }
      const int jm = j + (mi >> 1);            // column group of this lane's matrix row
      stmatrix_x4(arow + (uint32_t)((jm >> 3) & 1) * kFragBox + (uint32_t)(((jm & 7) ^ rr) << 4), hv[0], hv[1], hv[2], hv[3]);
    }
    fence_proxy_async();
    named_bar(1 + wg, 128);
    if (t == 0) {
      tma_store_3d(&p.y_store, buf, col0 + 128 * hf, 0, r);
      tma_store_3d(&p.y_store, buf + kFragBox, col0 + 128 * hf + 64, 0, r);
      bulk_commit_group();
    }
  }
}

// ------------------------------------------------------------------------------------------------
// the kernel
// ------------------------------------------------------------------------------------------------
constexpr int kATile = 128 * 128;   // 128 rows x 64 fp16
constexpr int kBTile = 128 * 128;   // one TMA box of B: 128 output columns x 64 fp16
constexpr int kEpiPitch = 65;       // floats per staged accumulator row: row-wise reads hit 32 distinct banks
constexpr int kEpiBytes = 64 * kEpiPitch * 4;
constexpr int kMaxSmemPerBlock = 232448;   // sm_90 opt-in limit, static + dynamic

template <int PASSES, bool SEGMENTED, int AMODE>
struct GemmCfg {
  static constexpr int NOP = PASSES == 3 ? 2 : 1;
  static constexpr int THREADS = AMODE == AMODE_GATHER ? 512 : 384;
  // Output columns per tile.  The 1-pass unsegmented 384-thread kernels (the window-map conv1 among them) use 128x256
  // tiles (m64n256k16, 128 accumulators per consumer thread): half the shared-memory operand reads per MAC, half the
  // A re-streaming and half the epilogues of 128x128.  Everything else stays at 128:
  //   3-pass and segmented kernels: their fp32 totals do not fit beside 128 accumulators;
  //   the 512-thread gather conv1 (AMODE_GATHER): ptxas needs each instruction's operands to fit the kernel-wide
  //   register target, 65536 / 512 = 128, whatever setmaxnreg grants, so m64n256k16 does not compile there; two
  //   m64n128k16 per k16 slice do, but the epilogue beside 128 accumulators then spills at every producer /
  //   A-operand / consumer split that fits their 4 x 128 registers per thread slot.
  static constexpr int BN = PASSES == 1 && !SEGMENTED && THREADS == 384 ? 256 : 128;
  static constexpr int B_BYTES = BN * 128;                 // BN rows x 64 fp16, BN / 128 TMA boxes back to back
  static constexpr int STAGE_BYTES = NOP * (kATile + B_BYTES);
  // 48 KB 256-wide stages: 4 fit beside the epilogue staging (6 of the 32 KB 1-pass 128-wide ones)
  static constexpr int STAGES = PASSES == 3 ? 3 : (THREADS == 512 ? 4 : (BN == 256 ? 4 : 6));
  static constexpr int SMEM = STAGES * STAGE_BYTES + 2 * kEpiBytes + 1024;
  static constexpr int FG = AMODE == AMODE_GATHER ? 16 : 1;
  static constexpr int STATIC_SMEM = 3 * STAGES * 8 + 2 * 2 * FG * FG * 4 + 2 * 4 * 4;   // barriers, fg_dinv, fg_org
  static_assert(SMEM + STATIC_SMEM <= kMaxSmemPerBlock, "shared memory over the per-block limit");
  // Per-thread registers after setmaxnreg.  The kernel starts with 65536 / THREADS (rounded down to 8) everywhere;
  // the producer warpgroup gives most of its share to the two consumer warpgroups (BN / 2 accumulators, plus 64
  // totals when SEGMENTED); the gather warpgroup (AMODE_GATHER, 512 threads) keeps what it needs.  The window-map
  // fix-up warps (AMODE_WINDOW) are warps 1-3 of the producer warpgroup and run at the producer's 24.
  static constexpr int LAUNCH_REGS = (65536 / THREADS) & ~7;
  // 256-wide: 240 per consumer (the 1-pass correlation epilogue spills at 232 beside 128 accumulators).
  static constexpr int PRODUCER_REGS = THREADS == 512 || BN == 256 ? 24 : 40;
  static constexpr int AUX_REGS = THREADS == 512 ? 128 : 0;
  static constexpr int CONSUMER_REGS = THREADS == 512 ? 176 : (BN == 256 ? 240 : 232);
  // setmaxnreg.inc only gets what other warpgroups of the CTA released from its launch allocation (LAUNCH_REGS per
  // thread), not the rest of the register file: a larger sum leaves the consumers blocked in setmaxnreg forever
  static_assert(PRODUCER_REGS + 2 * CONSUMER_REGS + AUX_REGS <= THREADS / 128 * LAUNCH_REGS, "register budget overcommitted");
  static_assert(PRODUCER_REGS <= LAUNCH_REGS && CONSUMER_REGS >= LAUNCH_REGS && AUX_REGS <= LAUNCH_REGS, "setmaxnreg direction");
};

__device__ __forceinline__ int fg_clamp(int v, int ds, int full) {   // ((x+dx)//ds).clamp(0, full//ds-1)
  if (v < 0) return 0;
  const int q = v / ds, m = full / ds - 1;
  return q < m ? q : m;
}

// AMODE_WINDOW: window origin of patch n in padded map coordinates: window pixel (wy, wx) lives at (oy + wy, ox + wx).
// Truncation = `.long()` (networks/utils.py:19); clamping the origin to [-7, W + 8] leaves every clamped window
// pixel unchanged (beyond that all of them sit on the border pixel) and keeps the boxes inside the padded map.
__device__ __forceinline__ int window_origin(const WindowMaps& wm, int n, int j) {
  int v;
  if (wm.is_float) v = (int)reinterpret_cast<const float*>(wm.matches)[(size_t)n * 4 + j];
  else v = (int)reinterpret_cast<const long long*>(wm.matches)[(size_t)n * 4 + j];
  const int lim = (j & 1) ? wm.H[j >> 1] : wm.W[j >> 1];
  v = v < -7 ? -7 : (v > lim + 8 ? lim + 8 : v);
  return v - 8 + kMapPad;
}

// AMODE_WINDOW: the matches row of patch slot s; past the end (odd patch counts) any valid row, the epilogue discards it
__device__ __forceinline__ int window_row(const WindowShare& ws, int s, int n_units) {
  if (s >= n_units) s = 0;
  return ws.slot_row != nullptr ? __ldg(ws.slot_row + s) : s;
}

// Tile = 128 rows x BN columns (see GemmCfg); K chunk 64 (one 128-byte swizzle row)
// per pipeline stage.
// Warpgroup 0: warp 0 is the TMA producer.  Warpgroups 1 and 2: wgmma consumers, rows 0..63 and 64..127, fp32
// accumulators in registers; their epilogue stages the accumulators through shared memory so that every epilogue
// thread owns one tile row (32 consecutive columns per piece), the layout epilogue_piece expects.
// conv1 (1-pass only) can take its A operand from elsewhere than a materialised patch tensor:
//   AMODE_GATHER  a fourth warpgroup gathers, normalises and converts the patch windows straight into the swizzled
//                 stage (select_local_patch_feats + patch L2Normalize, networks/utils.py:4-36,
//                 networks/patch2pix.py:173-178);
//   AMODE_WINDOW  the A boxes come by TMA from the per-image window maps (one strided box {64 ch, 8 px stride 2, 8 px
//                 stride 2} per patch and tap) and the rgb k-step from the im2col tensor window_rgb_kernel writes.
//                 Warps 1-3 of the producer warpgroup restore the conv's zero padding -- window pixel -1 must
//                 contribute 0, but the box holds the neighbouring image pixel there -- by zeroing the affected rows.
// Both A modes produce bit-identical operands and the same MMA sequence per output element.
// PASSES = 3: lo*hi + hi*lo + hi*hi into one accumulator.  SEGMENTED: the accumulator restarts every `seg_len`
// k-steps and each partial sum is added to fp32 register totals with round-to-nearest, which bounds the
// accumulator-rounding drift of long K chains.
template <int PASSES, bool SEGMENTED, int EPI, int AMODE>
__global__ void __launch_bounds__(GemmCfg<PASSES, SEGMENTED, AMODE>::THREADS, 1) umma_gemm_kernel(const __grid_constant__ UmmaGemmParams p) {
  static_assert(AMODE == AMODE_TMA || (PASSES == 1 && !SEGMENTED && EPI == EPI_CONV1), "fused A operand: conv1, 1-pass only");
  using Cfg = GemmCfg<PASSES, SEGMENTED, AMODE>;
  constexpr int STAGES = Cfg::STAGES, NOP = Cfg::NOP, STAGE_BYTES = Cfg::STAGE_BYTES;
  constexpr int BN = Cfg::BN, B_BYTES = Cfg::B_BYTES, NACC = BN / 2;
  // 256-wide conv1 / conv2: p.frag_epi selects the fragment epilogues (conv1_frag / conv2_frag) over the staged one.
  // They reuse the staging area: conv1 one 2-box buffer per warpgroup; conv2 a [4][256] max array per warpgroup and the
  // CTA's scale and bias (4 KB), which do not fit beside conv1's buffers.
  constexpr bool FRAG = BN == 256 && (EPI == EPI_CONV1 || EPI == EPI_CONV2);
  static_assert(2 * kFragBox * 2 <= 2 * kEpiBytes && 3 * 1024 * 4 <= 2 * kEpiBytes && (STAGES * STAGE_BYTES) % 1024 == 0,
                "fragment epilogue buffers");

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  float* epi_smem = reinterpret_cast<float*>(smem + STAGES * STAGE_BYTES);
  __shared__ __align__(8) uint64_t full_bar[STAGES];    // TMA bytes landed (+ gather warps in AMODE_GATHER)
  __shared__ __align__(8) uint64_t ready_bar[STAGES];   // AMODE_WINDOW: the fix-up warps are done with the stage
  __shared__ __align__(8) uint64_t empty_bar[STAGES];   // both consumer warpgroups are done reading the stage
  constexpr int FG = Cfg::FG;
  __shared__ float fg_dinv[2][2][FG][FG];               // act_scale / patch norm per (patch, image, window pixel)
  __shared__ int fg_org[2][4];                          // window origins (x1,y1,x2,y2) - 8

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  int m_tiles = p.m_tiles;
  int n_units = p.epi.n_patches;
  if (p.d_units != nullptr) {
    n_units = __ldg(p.d_units);
    m_tiles = (n_units + p.a_units_per_tile - 1) / p.a_units_per_tile;
  }
  const int n_col_tiles = p.n_tiles * (256 / BN);          // BN-column tiles
  const int total_tiles = m_tiles * n_col_tiles;
  const int nsteps = p.nsteps;
  const int seg_len = SEGMENTED ? p.seg_len : nsteps;
  // WindowShare: tiles from split_tile on are of class 1 and read steps[class_steps ..] (producer and fix-up warps only:
  // both classes run nsteps k-steps, so every role walks the same stage sequence)
  int split_tile = total_tiles, split_unit = 0;
  if (AMODE == AMODE_WINDOW && p.ws.d_split != nullptr) {
    split_tile = __ldg(p.ws.d_split);
    split_unit = __ldg(p.ws.d_split + 1);
  }

  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&p.b_hi);
    if (AMODE == AMODE_TMA) tma_prefetch_desc(&p.a_main_hi);
    if (AMODE == AMODE_WINDOW) {
      tma_prefetch_desc(&p.wm.map[0]);
      tma_prefetch_desc(&p.wm.map[1]);
      tma_prefetch_desc(&p.a_rgb_hi);
    }
    if (PASSES == 3) {
      tma_prefetch_desc(&p.a_main_lo);
      tma_prefetch_desc(&p.b_lo);
    }
    if (FRAG && EPI == EPI_CONV1 && p.frag_epi) tma_prefetch_desc(&p.y_store);
  }
  if (warp == 1 && lane == 0) {
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(&full_bar[i], AMODE == AMODE_GATHER ? 5 : 1);
      mbar_init(&ready_bar[i], 3);
      mbar_init(&empty_bar[i], 2);
    }
    fence_barrier_init();
  }
  __syncthreads();

  const int wgi = warpgroup_index();
  if (wgi == 0) {
    // ===================== TMA producer (warp 0, one thread) =====================
    setmaxnreg_dec<Cfg::PRODUCER_REGS>();
    if (warp == 0 && lane == 0) {
      int it = 0;
      // B tile of a stage: BN / 128 boxes of 128 rows into consecutive 16 KB, one descriptor spans them
      auto load_b = [&](const CUtensorMap* map, uint64_t* bar, uint8_t* dst, int bk, int brow) {
#pragma unroll
        for (int h = 0; h < BN / 128; ++h) tma_load_2d(map, bar, dst + h * kBTile, bk, brow + h * 128);
      };
      for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
        const int m_tile = tile / n_col_tiles, brow = (tile - m_tile * n_col_tiles) * BN;
        const int a4 = m_tile * p.a_units_per_tile;
        const int kofs = m_tile < split_tile ? 0 : p.ws.class_steps;
        if (p.trace != nullptr) {
          mbar_wait(&empty_bar[it % STAGES], ((uint32_t)(it / STAGES) & 1u) ^ 1u);
          p.trace[(size_t)tile * kTraceStamps] = globaltimer();
        }
        if (AMODE == AMODE_WINDOW && p.ws.part_in != nullptr) {
          // continuation: the tile's partial sums go to L2 now, so that its epilogue does not wait on HBM
#pragma unroll 1
          for (int pp = 0; pp < 2; ++pp)
            if (m_tile * 2 + pp < n_units)
              bulk_prefetch_l2(p.ws.part_in + part_offset(part_unit(m_tile * 2 + pp, 2 * split_tile, split_unit), 0, brow),
                               64 * 256 * 4);
        }
        int o[2][4];
        if (AMODE == AMODE_WINDOW) {
#pragma unroll
          for (int pp = 0; pp < 2; ++pp) {
            const int row = window_row(p.ws, m_tile * 2 + pp, n_units);
#pragma unroll
            for (int j = 0; j < 4; ++j) o[pp][j] = window_origin(p.wm, row, j);
          }
        }
        for (int ks = 0; ks < nsteps; ++ks, ++it) {
          const int s = it % STAGES;
          mbar_wait(&empty_bar[s], ((uint32_t)(it / STAGES) & 1u) ^ 1u);
          const KStep k = p.steps[ks + kofs];  // param space (constant bank)
          uint8_t* st = smem + (size_t)s * STAGE_BYTES;
          if (AMODE == AMODE_GATHER) {
            mbar_expect_tx(&full_bar[s], B_BYTES);
            load_b(&p.b_hi, &full_bar[s], st + kATile, k.bk, brow);
          } else if (AMODE == AMODE_WINDOW) {
            mbar_expect_tx(&full_bar[s], STAGE_BYTES);
            load_b(&p.b_hi, &full_bar[s], st + kATile, k.bk, brow);
            if (k.kind == 0) {
              const int ty = (k.plane & 2) ? 1 : (k.y < 0 ? 0 : 2), tx = (k.plane & 1) ? 1 : (k.x < 0 ? 0 : 2);
              const int chunk = k.c0 >> 6, si = chunk >> 2, c0 = (chunk & 3) * 64;
#pragma unroll
              for (int pp = 0; pp < 2; ++pp)
                tma_load_3d(&p.wm.map[si], &full_bar[s], st + pp * 8192, c0, o[pp][2 * si] - 1 + tx, o[pp][2 * si + 1] - 1 + ty);
            } else {
              tma_load_5d(&p.a_rgb_hi, &full_bar[s], st, 0, 0, 0, 0, a4);
            }
          } else {
            mbar_expect_tx(&full_bar[s], STAGE_BYTES);
            if (k.kind == 0) {
              tma_load_5d(&p.a_main_hi, &full_bar[s], st, k.c0, k.x, k.y, k.plane, a4);
              if (PASSES == 3) tma_load_5d(&p.a_main_lo, &full_bar[s], st + kATile, k.c0, k.x, k.y, k.plane, a4);
            } else {
              tma_load_5d(&p.a_rgb_hi, &full_bar[s], st, 0, 0, 0, 0, a4);
              if (PASSES == 3) tma_load_5d(&p.a_rgb_lo, &full_bar[s], st + kATile, 0, 0, 0, 0, a4);
            }
            load_b(&p.b_hi, &full_bar[s], st + NOP * kATile, k.bk, brow);
            if (PASSES == 3) load_b(&p.b_lo, &full_bar[s], st + NOP * kATile + B_BYTES, k.bk, brow);
          }
        }
      }
    } else if (AMODE == AMODE_WINDOW && warp > 0) {
      // ===================== zero-padding fix-up (warps 1-3) =====================
      // Taps with tx = 0 (ty = 0) read window column (row) -1 for output column ox = 0 (row oy = 0), which the conv
      // pads with zeros: those 16 tile rows (8 per patch) are cleared after the TMA bytes land.  Work item i of the
      // 2 x 16 candidate rows x 8 16-byte chunks: rows 0..15 are the ox = 0 rows, 16..31 the oy = 0 rows.
      const int t = threadIdx.x - 32;                  // 0..95
      int it = 0;
      for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
        const int kofs = tile / n_col_tiles < split_tile ? 0 : p.ws.class_steps;
        for (int ks = 0; ks < nsteps; ++ks, ++it) {
          const int s = it % STAGES;
          // every fix-up warp follows every stage (wait + arrive): parity waits are only valid within one ring
          // revolution, so no warp may run ahead of -- or fall behind -- the pipeline
          mbar_wait(&full_bar[s], (uint32_t)(it / STAGES) & 1u);
          const KStep k = p.steps[ks + kofs];
          const bool zx = k.kind == 0 && !(k.plane & 1) && k.x < 0, zy = k.kind == 0 && !(k.plane & 2) && k.y < 0;
          if (zx || zy) {
            uint8_t* st = smem + (size_t)s * STAGE_BYTES;
            for (int i = t; i < 256; i += 96) {
              const int j = i >> 3, pp = (j >> 3) & 1, r8 = j & 7;
              const int row = pp * 64 + (j < 16 ? r8 * 8 : r8);
              if (j < 16 ? zx : zy) *reinterpret_cast<uint4*>(st + row * 128 + (i & 7) * 16) = make_uint4(0, 0, 0, 0);
            }
            fence_proxy_async();
          }
          __syncwarp();
          if (lane == 0) mbar_arrive(&ready_bar[s]);
        }
      }
    }
  } else if (wgi < 3) {
    // ===================== wgmma consumers + epilogue (warpgroups 1 and 2) =====================
    setmaxnreg_inc<Cfg::CONSUMER_REGS>();
    const int wg = wgi - 1, wl = warp & 3;
    const bool leader = threadIdx.x % 128 == 0;    // arrives on empty_bar for the warpgroup
    uint64_t* ready = AMODE == AMODE_WINDOW ? ready_bar : full_bar;
    float* stg = epi_smem + wg * (64 * kEpiPitch);
    if (FRAG && EPI == EPI_CONV2 && p.frag_epi) {   // scale, bias -> epi_smem[2048 ..), past both warpgroups' max arrays
      const int t = threadIdx.x - 128;
      for (int i = t; i < 1024; i += 256) epi_smem[2048 + i] = i < 512 ? __ldg(p.epi.scale + i) : __ldg(p.epi.bias + i - 512);
      named_bar(4, 256);
    }
    float acc[NACC];
    float tot[SEGMENTED ? NACC : 1];
    int it = 0;
    for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
      const int m_tile = tile / n_col_tiles, col0 = (tile - m_tile * n_col_tiles) * BN;
      if (SEGMENTED) {
#pragma unroll
        for (int i = 0; i < NACC; ++i) tot[i] = 0.f;
      }
      unsigned long long* tr = p.trace != nullptr && threadIdx.x == 128 ? p.trace + (size_t)tile * kTraceStamps : nullptr;
      if (p.trace != nullptr) {   // the loop's own wait for this stage then returns at once
        if (tr != nullptr) tr[1] = globaltimer();
        mbar_wait(&ready[it % STAGES], (uint32_t)(it / STAGES) & 1u);
        if (tr != nullptr) tr[2] = globaltimer();
      }
      // Each k-step's MMAs are one wgmma group.  wait_group 1 after issuing step ks retires step ks - 1, whose stage
      // is then released, so the tensor core always has the next group queued.  An interior segment end drains the
      // pipe (wait_group 0) to add the partial sum and releases both stages; the tile's last step drains after the loop.
      for (int ks = 0; ks < nsteps; ++ks, ++it) {
        const int s = it % STAGES;
        mbar_wait(&ready[s], (uint32_t)(it / STAGES) & 1u);
        const uint32_t sa = smem_u32(smem + (size_t)s * STAGE_BYTES);
        const uint64_t a_hi = make_sw128_desc(sa + wg * 8192);
        const uint64_t b_hi = make_sw128_desc(sa + NOP * kATile);
        uint32_t accf = (ks % seg_len) == 0 ? 0u : 1u;
        wgmma_fence();
        if (PASSES == 3) {
          const uint64_t a_lo = make_sw128_desc(sa + kATile + wg * 8192);
          const uint64_t b_lo = make_sw128_desc(sa + NOP * kATile + B_BYTES);
#pragma unroll
          for (int kk = 0; kk < 4; ++kk) {
            wgmma_f16<BN>(acc, a_lo + 2 * kk, b_hi + 2 * kk, accf);
            accf = 1u;
          }
#pragma unroll
          for (int kk = 0; kk < 4; ++kk) wgmma_f16<BN>(acc, a_hi + 2 * kk, b_lo + 2 * kk, 1u);
        }
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {
          wgmma_f16<BN>(acc, a_hi + 2 * kk, b_hi + 2 * kk, accf);
          accf = 1u;
        }
        wgmma_commit();
        // both conditions depend on the k-step counter and kernel parameters only: uniform across the warpgroup
        const bool seg_end = SEGMENTED && ((ks + 1) % seg_len) == 0 && (ks + 1) < nsteps;
        const bool prev_pending = SEGMENTED ? (ks % seg_len) != 0 : ks != 0;   // step ks - 1 is not yet released
        if (seg_end) {
          wgmma_wait<0>();
          wgmma_fence_regs<NACC>(acc);
#pragma unroll
          for (int i = 0; i < NACC; ++i) tot[i] += acc[i];
        } else {
          wgmma_wait<1>();
        }
        mbar_arrive_if(&empty_bar[(s + STAGES - 1) % STAGES], leader && prev_pending);
        mbar_arrive_if(&empty_bar[s], leader && seg_end);
      }
      if (tr != nullptr) tr[3] = globaltimer();
      wgmma_wait<0>();
      wgmma_fence_regs<NACC>(acc);
      if (tr != nullptr) tr[4] = globaltimer();
      mbar_arrive_if(&empty_bar[(it + STAGES - 1) % STAGES], leader);   // the tile's last k-step
      if (SEGMENTED) {
#pragma unroll
        for (int i = 0; i < NACC; ++i) tot[i] += acc[i];
      }
      if (FRAG && p.frag_epi) {
        if (EPI == EPI_CONV2)
          conv2_frag(p.epi, acc, m_tile * 2 + wg, n_units, col0, reinterpret_cast<uint32_t*>(epi_smem) + wg * 1024,
                     epi_smem + 2 * 1024, wg);
        else
          conv1_frag<AMODE == AMODE_WINDOW>(p, acc, m_tile * 2 + wg, n_units, 2 * split_tile, split_unit, col0,
                                            reinterpret_cast<uint8_t*>(epi_smem) + wg * 2 * kFragBox);
      } else {
        const float* res = SEGMENTED ? tot : acc;
        // fragment -> row-major staging, 64 columns at a time; then one row per thread
        const int fr = 16 * wl + (lane >> 2), fc = 2 * (lane & 3);
        const int er = (wl & 1) * 32 + lane, ec = (wl >> 1) * 32;
#pragma unroll
        for (int c64 = 0; c64 < BN / 64; ++c64) {
          named_bar(1 + wg, 128);                 // the previous piece has been read
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const float* d = res + 4 * (c64 * 8 + j);
            float* o = stg + fr * kEpiPitch + 8 * j + fc;
            o[0] = d[0];
            o[1] = d[1];
            o[8 * kEpiPitch] = d[2];
            o[8 * kEpiPitch + 1] = d[3];
          }
          named_bar(1 + wg, 128);
          if (AMODE == AMODE_WINDOW && (p.ws.part_out != nullptr || p.ws.part_in != nullptr)) {
            share_piece(p.ws, 2 * split_tile, split_unit, n_units, m_tile, wg * 64 + er, col0 + c64 * 64 + ec,
                        stg + er * kEpiPitch + ec);
            if (p.ws.part_out != nullptr) continue;   // prefix launch: no BN, no y_hi, no pooled zeroing
          }
          float v[32];
#pragma unroll
          for (int i = 0; i < 32; ++i) v[i] = stg[er * kEpiPitch + ec + i];
          epilogue_piece<EPI, AMODE == AMODE_WINDOW>(p.epi, p.ws, n_units, m_tile, wg * 64 + er, col0 + c64 * 64 + ec, v);
        }
      }
      if (tr != nullptr) {
        tr[5] = globaltimer();
        tr[6] = blockIdx.x + 1;
      }
    }
    if (FRAG && EPI == EPI_CONV1 && p.frag_epi && threadIdx.x % 128 == 0) bulk_wait_group<0>();   // the last stores are complete
  } else if (AMODE == AMODE_GATHER) {
    // ===================== fused A-operand producers (warpgroup 3) =====================
    if constexpr (Cfg::AUX_REGS < Cfg::LAUNCH_REGS) setmaxnreg_dec<Cfg::AUX_REGS>();
    // 8 lanes per tile row (8 channels = 16 B each), 16 rows per pass, 8 passes per k-step.  Warps drift across
    // pipeline stages independently, which hides the L2 latency of the gathers.
    const int ptid = threadIdx.x - 384;
    const int l8 = ptid & 7, r16 = ptid >> 3;
    const FusedGather& g = p.fg;
    int it = 0;
    for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
      const int m_tile = tile / n_col_tiles;
      named_bar(3, 128);   // nobody still reads the previous tile's tables
      if (ptid < 8) {
        const int pp = ptid >> 2, j = ptid & 3;
        const int n = m_tile * 2 + pp;
        int v = 0;
        if (n < n_units) {
          if (g.is_float)
            v = (int)reinterpret_cast<const float*>(g.matches)[(size_t)n * 4 + j];   // .long(): truncation
          else
            v = (int)reinterpret_cast<const long long*>(g.matches)[(size_t)n * 4 + j];
        }
        fg_org[pp][j] = v - 8;
      }
      named_bar(3, 128);
      for (int i = ptid; i < 1024; i += 128) {
        const int pp = i >> 9, si = (i >> 8) & 1, wy = (i >> 4) & 15, wx = i & 15;
        const int X = fg_org[pp][2 * si] + wx, Y = fg_org[pp][2 * si + 1] + wy;
        float t = 0.f;
#pragma unroll
        for (int l = 0; l < 4; ++l) {
          const int ds = 1 << l;
          const int xi = fg_clamp(X, ds, g.W[si]), yi = fg_clamp(Y, ds, g.H[si]);
          t += __ldg(g.nsq[si][l] + (size_t)yi * (g.W[si] / ds) + xi);
        }
        fg_dinv[pp][si][wy][wx] = (m_tile * 2 + pp < n_units) ? __fdiv_rn(kActScale, sqrtf(t + 1e-6f)) : 0.f;
      }
      named_bar(3, 128);
      for (int ks = 0; ks < nsteps; ++ks, ++it) {
        const int s = it % STAGES;
        const uint32_t ph = (uint32_t)(it / STAGES) & 1u;
        const KStep k = p.steps[ks];
        uint8_t* at = smem + (size_t)s * STAGE_BYTES;
        if (k.kind == 0) {
          const int ty = (k.plane & 2) ? 1 : (k.y < 0 ? 0 : 2), tx = (k.plane & 1) ? 1 : (k.x < 0 ? 0 : 2);
          const int chunk = k.c0 >> 6, si = chunk >> 2, jj = chunk & 3;
          const int lvl = jj == 0 ? 0 : (jj == 1 ? 1 : 2);
          const int sh = lvl + 1, C = lvl == 2 ? 128 : 64;
          const int coff = (jj == 3 ? 64 : 0) + l8 * 8;
          const __half* fmap = g.nhwc16[si][lvl];
          const float* nsq = g.nsq[si][lvl + 1];
          const int wl = g.W[si] >> sh, hl = g.H[si] >> sh;
          uint4 vals[8];
          float sc[8];
#pragma unroll
          for (int ps = 0; ps < 8; ++ps) {               // phase 1: every load in flight before any use
            const int row = ps * 16 + r16;
            const int pp = row >> 6, wy = 2 * ((row >> 3) & 7) - 1 + ty, wx = 2 * (row & 7) - 1 + tx;
            const int X = fg_org[pp][2 * si] + wx, Y = fg_org[pp][2 * si + 1] + wy;
            const int xi = X < 0 ? 0 : min(X >> sh, wl - 1), yi = Y < 0 ? 0 : min(Y >> sh, hl - 1);
            const int px = yi * wl + xi;
            vals[ps] = __ldg(reinterpret_cast<const uint4*>(fmap + (size_t)px * C + coff));
            // undo the per-level normalisation; window pixel -1 = conv zero padding
            const float dv = (wy >= 0 && wx >= 0) ? fg_dinv[pp][si][wy & 15][wx & 15] : 0.f;
            sc[ps] = dv * sqrtf(__ldg(nsq + px) + 1e-30f);
          }
          mbar_wait(&empty_bar[s], ph ^ 1u);
#pragma unroll
          for (int ps = 0; ps < 8; ++ps) {               // phase 2: scale, convert, swizzled store
            const int row = ps * 16 + r16;
            __half2* h2 = reinterpret_cast<__half2*>(&vals[ps]);
#pragma unroll
            for (int q = 0; q < 4; ++q) {
              const float2 f = __half22float2(h2[q]);
              h2[q] = __floats2half2_rn(f.x * sc[ps], f.y * sc[ps]);
            }
            *reinterpret_cast<uint4*>(at + row * 128 + ((l8 ^ (row & 7)) << 4)) = vals[ps];
          }
        } else {
          // rgb im2col chunk: k = tap*6 + img*3 + ch (54 used)
          mbar_wait(&empty_bar[s], ph ^ 1u);
#pragma unroll 1
          for (int ps = 0; ps < 8; ++ps) {
            const int row = ps * 16 + r16;
            const int pp = row >> 6, oy = (row >> 3) & 7, ox = row & 7;
            __align__(16) __half hv[8];
#pragma unroll
            for (int i = 0; i < 8; ++i) {
              const int kk = l8 * 8 + i;
              float v = 0.f;
              if (kk < 54) {
                const int tap = kk / 6, r = kk - tap * 6;
                const int si = r / 3, ch = r - si * 3;
                const int wx = 2 * ox - 1 + tap % 3, wy = 2 * oy - 1 + tap / 3;
                if (wx >= 0 && wy >= 0) {
                  const int xi = fg_clamp(fg_org[pp][2 * si] + wx, 1, g.W[si]);
                  const int yi = fg_clamp(fg_org[pp][2 * si + 1] + wy, 1, g.H[si]);
                  v = __ldg(g.img[si] + ((size_t)ch * g.H[si] + yi) * g.W[si] + xi) * fg_dinv[pp][si][wy][wx];
                }
              }
              hv[i] = __float2half_rn(v);
            }
            *reinterpret_cast<uint4*>(at + row * 128 + ((l8 ^ (row & 7)) << 4)) = *reinterpret_cast<const uint4*>(hv);
          }
        }
        fence_proxy_async();            // generic-proxy stores -> visible to the tensor core (async proxy)
        __syncwarp();
        if (lane == 0) mbar_arrive(&full_bar[s]);
      }
    }
  }
}

// AMODE_WINDOW's rgb k-step: the im2col rows of every patch, [npad][64 output px][64] fp16 with k = tap*6 + img*3 + ch
// (54 used, rest zero), copied from the normalised rgb maps; window pixel -1 = conv zero padding, and the pad patch of
// an odd count is all zero.  One thread per output pixel (row of 128 bytes).
__global__ void __launch_bounds__(256) window_rgb_kernel(const __grid_constant__ WindowMaps wm, int n_units, int npad,
                                                         __half* __restrict__ out, const int* __restrict__ slot_row,
                                                         const int* __restrict__ d_count) {
  const int row = blockIdx.x * 256 + threadIdx.x;
  if (row >= npad * 64) return;
  const int n = row >> 6, oy = (row >> 3) & 7, ox = row & 7;
  if (d_count != nullptr) {
    n_units = __ldg(d_count);
    if (n >= n_units + (n_units & 1)) return;      // beyond the pad slot: no tile reads it
  }
  __align__(16) __half hv[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) hv[i] = __float2half_rn(0.f);
  if (n < n_units) {
    const int r = slot_row != nullptr ? __ldg(slot_row + n) : n;
#pragma unroll
    for (int si = 0; si < 2; ++si) {
      const int bx = window_origin(wm, r, 2 * si), by = window_origin(wm, r, 2 * si + 1);
      const int Wp = map_pitch(wm.W[si]);
#pragma unroll
      for (int tap = 0; tap < 9; ++tap) {
        const int wx = 2 * ox - 1 + tap % 3, wy = 2 * oy - 1 + tap / 3;
        if (wx >= 0 && wy >= 0) {
          const uint2 q = __ldg(reinterpret_cast<const uint2*>(wm.rgbn[si] + ((size_t)(by + wy) * Wp + bx + wx) * 4));
          const __half* hq = reinterpret_cast<const __half*>(&q);
          hv[tap * 6 + si * 3 + 0] = hq[0];
          hv[tap * 6 + si * 3 + 1] = hq[1];
          hv[tap * 6 + si * 3 + 2] = hq[2];
        }
      }
    }
  }
  uint4* dst = reinterpret_cast<uint4*>(out + (size_t)row * 64);
#pragma unroll
  for (int c = 0; c < 8; ++c) dst[c] = reinterpret_cast<const uint4*>(hv)[c];
}

int launch_window_rgb(const WindowMaps& wm, int n, int npad, __half* out, cudaStream_t st, const int* slot_row,
                      const int* d_count) {
  P2P_REQUIRE(n >= 0 && npad >= n, "window rgb: bad patch count");
  if (npad == 0) return 0;
  window_rgb_kernel<<<(unsigned)cdiv(npad * 64, 256), 256, 0, st>>>(wm, n, npad, out, slot_row, d_count);
  P2P_LAUNCH_OK();
  return 0;
}

// Block-wide exclusive prefix sums of three counters per thread (1024 threads); tot receives the block totals.
__device__ __forceinline__ void block_scan3(const int (&v)[3], int (&ex)[3], int (&tot)[3], int (*s_warp)[32]) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  int inc[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    inc[c] = v[c];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int t = __shfl_up_sync(0xffffffffu, inc[c], o);
      if (lane >= o) inc[c] += t;
    }
    if (lane == 31) s_warp[c][wid] = inc[c];
  }
  __syncthreads();
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    int woff = 0, t = 0;
    for (int w = 0; w < 32; ++w) {
      const int x = s_warp[c][w];
      if (w < wid) woff += x;
      t += x;
    }
    ex[c] = woff + inc[c] - v[c];
    tot[c] = t;
  }
  __syncthreads();
}

// Half-group h (0: rows 8g..8g+3, compared on image 2; 1: rows 8g+4..8g+7, compared on image 1) of a complete group
// is shared when its four window origins are equal.  Single block, one thread per group, order-preserving.
__global__ void __launch_bounds__(1024) window_share_classify_kernel(const __grid_constant__ WindowMaps wm, int n,
                                                                     int* __restrict__ prefix, int* __restrict__ cont,
                                                                     int* __restrict__ unsh, int* __restrict__ cnt,
                                                                     int* __restrict__ shared_out) {
  __shared__ int s_warp[3][32];
  __shared__ int s_base[3];   // A half-groups, B half-groups, unshared rows so far
  __shared__ int s_na;
  const int tid = threadIdx.x, groups = (n + 7) / 8;
  auto shared_half = [&](int g, int h) {
    if (8 * g + 8 > n) return 0;
    const int si = 1 - h, r0 = 8 * g + 4 * h;
    const int x = window_origin(wm, r0, 2 * si), y = window_origin(wm, r0, 2 * si + 1);
    for (int i = 1; i < 4; ++i)
      if (window_origin(wm, r0 + i, 2 * si) != x || window_origin(wm, r0 + i, 2 * si + 1) != y) return 0;
    return 1;
  };
  if (tid == 0) s_na = s_base[0] = s_base[1] = s_base[2] = 0;
  __syncthreads();
  int na = 0;
  for (int g = tid; g < groups; g += 1024) na += shared_half(g, 0);
  atomicAdd(&s_na, na);
  __syncthreads();
  const int nA = s_na, ubase = nA + (nA & 1);
  for (int g0 = 0; g0 < groups; g0 += 1024) {
    const int g = g0 + tid;
    int v[3] = {0, 0, 0};
    if (g < groups) {
      v[0] = shared_half(g, 0);
      v[1] = shared_half(g, 1);
      v[2] = min(8, n - 8 * g) - 4 * (v[0] + v[1]);
    }
    int ex[3], tot[3];
    block_scan3(v, ex, tot, s_warp);
    if (g < groups) {
      const int ia = s_base[0] + ex[0], ib = s_base[1] + ex[1];
      int iu = s_base[2] + ex[2];
      if (v[0]) {
        prefix[ia] = 8 * g;
        for (int i = 0; i < 4; ++i) cont[4 * ia + i] = 8 * g + i;
      }
      if (v[1]) {
        prefix[ubase + ib] = 8 * g + 4;
        for (int i = 0; i < 4; ++i) cont[4 * (nA + ib) + i] = 8 * g + 4 + i;
      }
      for (int r = 8 * g; r < min(8 * g + 8, n); ++r)
        if (!(r - 8 * g < 4 ? v[0] : v[1])) unsh[iu++] = r;
    }
    __syncthreads();
    if (tid == 0)
      for (int c = 0; c < 3; ++c) s_base[c] += tot[c];
    __syncthreads();
  }
  if (tid == 0) {
    const int nB = s_base[1];
    if (nA & 1) prefix[nA] = prefix[nA - 1];   // pad slot: computed, never read
    cnt[0] = ubase + nB;
    cnt[1] = ubase / 2;
    cnt[2] = 0;
    cnt[3] = 4 * (nA + nB);
    cnt[4] = 2 * nA;
    cnt[5] = ubase;
    cnt[6] = s_base[2];
    cnt[7] = 0;
    if (shared_out != nullptr) *shared_out = 4 * (nA + nB);
  }
}

int launch_window_share_classify(const WindowMaps& wm, int n, int* prefix, int* cont, int* unsh, int* cnt, int* shared_out,
                                 cudaStream_t st) {
  P2P_REQUIRE(n >= 0, "window share: bad row count");
  window_share_classify_kernel<<<1, 1024, 0, st>>>(wm, n, prefix, cont, unsh, cnt, shared_out);
  P2P_LAUNCH_OK();
  return 0;
}


// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
typedef CUresult (*PFN_tmapEncodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                        const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                        CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_tmapEncodeTiled get_encode_fn() {
  static PFN_tmapEncodeTiled fn = nullptr;
  if (fn == nullptr) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_tmapEncodeTiled>(p);
  }
  return fn;
}

// Encoded tensor maps are cached per host thread (keyed by base pointer + geometry): the scratch arenas are stable
// after the first pair of a given shape, so the ~36 descriptors of a refine stage are encoded once, not per launch.
namespace {
struct TmapKey {
  const void* base;
  int rank;
  uint64_t dims[5];
  uint64_t strides[4];
  uint32_t box[5];
  uint32_t es[5];
  bool operator==(const TmapKey& o) const { return memcmp(this, &o, sizeof(TmapKey)) == 0; }
};
struct TmapEntry {
  TmapKey key;
  CUtensorMap map;
};
constexpr int kTmapCacheSize = 128;
thread_local std::vector<TmapEntry> g_tmap_cache;
thread_local int g_tmap_next = 0;
}  // namespace

int make_tmap_fp16(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                   const uint32_t* box, const uint32_t* estrides) {
  TmapKey key;
  memset(&key, 0, sizeof(key));
  key.base = base;
  key.rank = rank;
  for (int i = 0; i < rank; ++i) { key.dims[i] = dims[i]; key.box[i] = box[i]; key.es[i] = estrides ? estrides[i] : 1; }
  for (int i = 0; i + 1 < rank; ++i) key.strides[i] = strides_bytes[i];
  for (const TmapEntry& e : g_tmap_cache)
    if (e.key == key) {
      *out = e.map;
      return 0;
    }
  PFN_tmapEncodeTiled fn = get_encode_fn();
  if (fn == nullptr) {
    set_last_error("cuTensorMapEncodeTiled is not available from the driver");
    return -2;
  }
  cuuint64_t gd[5];
  cuuint64_t gs[4];
  cuuint32_t bx[5], es[5];
  for (int i = 0; i < rank; ++i) {
    gd[i] = dims[i];
    bx[i] = box[i];
    es[i] = estrides ? estrides[i] : 1;
  }
  for (int i = 0; i + 1 < rank; ++i) gs[i] = strides_bytes[i];
  const CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, (cuuint32_t)rank, const_cast<void*>(base), gd, gs, bx, es,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_last_error("cuTensorMapEncodeTiled failed with CUresult " + std::to_string((int)r));
    return -2;
  }
  if ((int)g_tmap_cache.size() < kTmapCacheSize) {
    g_tmap_cache.push_back(TmapEntry{key, *out});
  } else {
    g_tmap_cache[g_tmap_next] = TmapEntry{key, *out};
    g_tmap_next = (g_tmap_next + 1) % kTmapCacheSize;
  }
  return 0;
}

template <int PASSES, bool SEGMENTED, int EPI, int AMODE = AMODE_TMA>
static int launch_one(const UmmaGemmParams& p, int num_sms, cudaStream_t st) {
  using Cfg = GemmCfg<PASSES, SEGMENTED, AMODE>;
  auto kern = umma_gemm_kernel<PASSES, SEGMENTED, EPI, AMODE>;
  const int total = p.m_tiles * p.n_tiles * (256 / Cfg::BN);
  const int grid = total < num_sms ? total : num_sms;
  P2P_ENSURE_SMEM(kern, Cfg::SMEM);
  kern<<<grid, Cfg::THREADS, Cfg::SMEM, st>>>(p);
  P2P_LAUNCH_OK();
  return 0;
}

template <int EPI>
static int launch_epi(const UmmaGemmParams& p, int passes, bool seg, int num_sms, cudaStream_t st) {
  if (passes == 3) return seg ? launch_one<3, true, EPI>(p, num_sms, st) : launch_one<3, false, EPI>(p, num_sms, st);
  return seg ? launch_one<1, true, EPI>(p, num_sms, st) : launch_one<1, false, EPI>(p, num_sms, st);
}

int launch_umma_gemm(const UmmaGemmParams& p, int epi, int passes, int num_sms, cudaStream_t st, int amode) {
  P2P_REQUIRE(passes == 1 || passes == 3, "umma gemm: passes must be 1 or 3");
  P2P_REQUIRE(p.nsteps > 0 && p.m_tiles > 0 && p.n_tiles > 0, "umma gemm: empty problem");
  const bool seg = p.seg_len > 0 && p.seg_len < p.nsteps;
  if (p.frag_epi) {
    P2P_REQUIRE((epi == EPI_CONV1 || epi == EPI_CONV2) && passes == 1 && !seg && amode != AMODE_GATHER,
                "umma gemm: the fragment epilogues serve the 256-wide conv1 / conv2 launches only");
    P2P_REQUIRE(epi == EPI_CONV2 || p.epi.y_lo == nullptr, "umma gemm: the fragment conv1 epilogue writes y_hi only");
  }
  if (amode != AMODE_TMA) {
    P2P_REQUIRE(epi == EPI_CONV1 && passes == 1 && !seg, "the fused A operand is available for 1-pass conv1 only");
    if (amode == AMODE_GATHER) return launch_one<1, false, EPI_CONV1, AMODE_GATHER>(p, num_sms, st);
    P2P_REQUIRE(amode == AMODE_WINDOW, "umma gemm: unknown A mode");
    return launch_one<1, false, EPI_CONV1, AMODE_WINDOW>(p, num_sms, st);
  }
  switch (epi) {
    case EPI_PLAIN: return launch_epi<EPI_PLAIN>(p, passes, seg, num_sms, st);
    case EPI_CONV1: return launch_epi<EPI_CONV1>(p, passes, seg, num_sms, st);
    case EPI_CONV2: return launch_epi<EPI_CONV2>(p, passes, seg, num_sms, st);
    case EPI_CORR: return launch_epi<EPI_CORR>(p, passes, seg, num_sms, st);
    case EPI_FC: return launch_epi<EPI_FC>(p, passes, seg, num_sms, st);
  }
  set_last_error("umma gemm: unknown epilogue");
  return -1;
}

}  // namespace p2p
