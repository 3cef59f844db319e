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
  CUtensorMap map[2];             // [H + 2 pad][W + 2 pad][256] fp16 per image; box = 64 ch x 8 (stride 2) x 8 (stride 2)
  const __half* rgbn[2];          // [H + 2 pad][W + 2 pad][4]
  int H[2], W[2];
  const void* matches;
  int is_float;
};

struct UmmaGemmParams {
  CUtensorMap a_main_hi, a_main_lo, a_rgb_hi, a_rgb_lo, b_hi, b_lo;
  KStep steps[kMaxKSteps];
  int nsteps;
  int m_tiles;           // 128-row tiles
  int n_tiles;           // 256-column blocks of B: one 256-column tile (1-pass unsegmented) or two 128-column tiles;
                         // B tensor maps have 128-row boxes
  int a_units_per_tile;  // step of the outermost A coordinate per m-tile (2 patches, or 128 rows)
  int seg_len;           // k-steps accumulated by the tensor core before a drain (0 / >= nsteps: whole K)
  const int* d_units;    // optional device count of A units (patches): m_tiles = ceil(*d_units / a_units_per_tile)
  UmmaEpilogue epi;
  FusedGather fg;        // AMODE_GATHER
  WindowMaps wm;         // AMODE_WINDOW
};

// estrides (optional): traversal strides; with stride s the box must be N * s to load N elements.
int make_tmap_fp16(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                   const uint32_t* box, const uint32_t* estrides = nullptr);
int launch_umma_gemm(const UmmaGemmParams& p, int epi, int passes, int num_sms, cudaStream_t st, int amode = AMODE_TMA);
// AMODE_WINDOW's rgb k-step operand: writes the [npad][64][64] fp16 im2col tensor of patches 0..n-1 (zeros beyond n)
int launch_window_rgb(const WindowMaps& wm, int n, int npad, __half* out, cudaStream_t st);

}  // namespace p2p
