// Parameters of the wgmma implicit-GEMM kernel (umma_gemm.cu).
#pragma once
#include <cuda.h>

#include "kernels.h"

namespace p2p {

enum { EPI_PLAIN = 0, EPI_CONV1 = 1, EPI_CONV2 = 2, EPI_CORR = 3, EPI_FC = 4 };
// where the A operand of a k-step comes from: TMA of a materialised tensor, gathered by producer warps (conv1), or TMA of
// the per-image window maps (conv1)
enum { AMODE_TMA = 0, AMODE_GATHER = 1, AMODE_WINDOW = 2 };
constexpr int kMaxKSteps = 96;
constexpr int kTraceStamps = 8;

struct UmmaEpilogue {
  // EPI_PLAIN / EPI_CORR output
  float* c;
  int ldc, m_rows, n_cols;
  float alpha;
  // EPI_CORR: pooled grid sizes and the argmax code
  uint8_t* code;
  int np1, np2;
  // EPI_CONV1 / EPI_CONV2
  const float* scale;   // [512]
  const float* bias;    // [512]
  float y_scale;
  __half* y_hi;
  __half* y_lo;
  float* pooled;
  int n_patches;
};

// conv1 with the patch gather fused into producer warps (AMODE_GATHER): the A tile of every k-step
// is built in shared memory straight from the channels-last fp16 pyramid copies.
struct FusedGather {
  const float* img[2];            // [3][H][W]
  const __half* nhwc16[2][3];     // level-normalised fp16 pyramid copies
  const float* nsq[2][4];         // per-level squared norms
  int H[2], W[2];
  const void* matches;            // [n][4] int64 or fp32
  int is_float;
};

// conv1 fed by strided TMA boxes of the per-image window maps (AMODE_WINDOW); the rgb k-step comes by TMA (a_rgb_hi)
// from the im2col tensor launch_window_rgb builds out of rgbn
struct WindowMaps {
  CUtensorMap map[2];             // [H + 2 pad][map_pitch(W)][256] fp16 per image; box = 64 ch x 8 (stride 2) x 8 (stride 2)
  const __half* rgbn[2];          // [H + 2 pad][map_pitch(W)][4]
  int H[2], W[2];
  const void* matches;
  int is_float;
};

// AMODE_WINDOW launches of the mid stage's shared anchor windows (api.cu, run_regressor); all zero: patch slot s is
// row s and every tile runs steps[0 .. nsteps).
//   prefix launch:       one slot per shared half-group, k-steps of the shared image only; the epilogue stores the raw
//                        fp32 accumulators to part_out[slot][2][64][256] (no BN, no y_hi, no pooled zeroing)
//   continuation launch: the half-groups' rows, k-steps of the other image + rgb; the epilogue adds
//                        part_in[unit][2][64][256] (4 consecutive slots per unit) before the BN, which the producer
//                        prefetches into L2 at the start of each tile
// Tiles from m-tile d_split[0] on are of class 1 and read steps[class_steps ..]; in the continuation the unit of
// class-1 slot s is d_split[1] + (s - 2 * d_split[0]) / 4, of class-0 slot s it is s / 4.
struct WindowShare {
  const int* slot_row;   // patch slot -> row of wm.matches (window origins) and of the conv1 outputs (null: the slot)
  const int* d_split;    // device {first class-1 m-tile, prefix unit of the first class-1 continuation slot}
  int class_steps;
  float* part_out;
  const float* part_in;
};

struct UmmaGemmParams {
  CUtensorMap a_main_hi, a_main_lo, a_rgb_hi, a_rgb_lo, b_hi, b_lo;
  // EPI_CONV1 with the fragment epilogue: TMA store of epi.y_hi as [rows][64 px][512 ch], box {64 ch, 64 px, 1 row}
  CUtensorMap y_store;
  KStep steps[kMaxKSteps];
  int nsteps;
  int m_tiles;           // 128-row tiles
  int n_tiles;           // 256-column blocks of B: one 256-column tile (1-pass unsegmented) or two 128-column tiles;
                         // B tensor maps have 128-row boxes
  int a_units_per_tile;  // step of the outermost A coordinate per m-tile (2 patches, or 128 rows)
  int seg_len;           // k-steps accumulated by the tensor core before a drain (0 / >= nsteps: whole K)
  // 1: the 256-wide (1-pass, unsegmented) EPI_CONV1 / EPI_CONV2 launches take their epilogue straight from the wgmma
  // fragments (conv1: the fp16 tile leaves by TMA store through y_store) instead of through the fp32 staging buffer;
  // both write identical bits
  int frag_epi;
  // optional per-tile phase trace (kTraceStamps %globaltimer stamps per tile, indexed by tile; zero-filled by the host):
  //   0 producer: the tile's first stage is free and its loads are about to issue
  //   1 consumer warpgroup 1: tile start   2 first stage ready   3 last k-step issued   4 accumulators drained
  //   5 epilogue done   6 blockIdx.x + 1
  unsigned long long* trace;
  const int* d_units;    // optional device count of A units (patches): m_tiles = ceil(*d_units / a_units_per_tile)
  UmmaEpilogue epi;
  FusedGather fg;        // AMODE_GATHER
  WindowMaps wm;         // AMODE_WINDOW
  WindowShare ws;        // AMODE_WINDOW
};

// estrides (optional): traversal strides; with stride s the box must be N * s to load N elements.
int make_tmap_fp16(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                   const uint32_t* box, const uint32_t* estrides = nullptr);
int launch_umma_gemm(const UmmaGemmParams& p, int epi, int passes, int num_sms, cudaStream_t st, int amode = AMODE_TMA);
// AMODE_WINDOW's rgb k-step operand: writes the [npad][64][64] fp16 im2col tensor of patches 0..n-1 (zeros beyond n).
// With slot_row / d_count (device): slot s < *d_count holds row slot_row[s]; an odd count's pad slot is zero and the
// slots beyond it are not written.
int launch_window_rgb(const WindowMaps& wm, int n, int npad, __half* out, cudaStream_t st, const int* slot_row = nullptr,
                      const int* d_count = nullptr);
// Anchor-window sharing of the mid stage's conv1 (WindowShare): over groups of 8 consecutive rows, half-group A (rows
// 8g..8g+3) is shared when its four image-2 window origins are equal, half-group B (8g+4..8g+7) when its four image-1
// origins are; a partial last group is never shared.  Writes, order-preserving:
//   prefix[]: A representatives, one pad slot if their count nA is odd, then B representatives (from slot ubase)
//   cont[]:   rows of the shared A half-groups, then those of the shared B half-groups
//   unsh[]:   every other row, ascending
//   cnt[8]:   {prefix slots, ubase / 2, 0, shared rows, 2 nA, ubase, unshared rows, 0}, ubase = nA rounded up to even
// prefix needs n / 4 + 2 entries, cont and unsh n each.  shared_out (optional): receives the shared-row count too.
int launch_window_share_classify(const WindowMaps& wm, int n, int* prefix, int* cont, int* unsh, int* cnt, int* shared_out,
                                 cudaStream_t st);

}  // namespace p2p
