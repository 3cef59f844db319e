// Internal launcher declarations shared by the translation units of libp2p_b200.so.
#pragma once
#include "common.cuh"

namespace p2p {

// ---- coarse.cu ---------------------------------------------------------------------------------
int launch_l2norm_perm(const float* in, float* out, int C, int h, int w, int ksize, cudaStream_t st);
// K-major fp16 hi/lo variant for the tensor-core correlation: out[q][c] = split(kActScale * f/|f|)
int launch_l2norm_perm_kmajor_pair(const float* in1, const float* in2, __half* hi1, __half* lo1, __half* hi2, __half* lo2,
                                   int C, int h1, int w1, int h2, int w2, int ksize, cudaStream_t st);
int launch_l2norm_perm_kmajor_pair_nhwc16(const __half* in1, const __half* in2, __half* hi1, __half* lo1, __half* hi2, __half* lo2,
                                          int C, int h1, int w1, int h2, int w2, int ksize, cudaStream_t st);
int launch_split_rows(const float* in, __half* hi, __half* lo, size_t n, float scale, cudaStream_t st);
int launch_delta_pack(const long long* di, const long long* dj, const long long* dk, const long long* dl, size_t n,
                      int ks, uint8_t* code, cudaStream_t st);
int launch_corr_pool_simt(const float* fa, const float* fb, int C, int n1, int n2, int ksize, float* out,
                          uint8_t* code, cudaStream_t st);
int launch_delta_unpack(const uint8_t* code, size_t n, int ks, long long* di, long long* dj, long long* dk,
                        long long* dl, cudaStream_t st);
// absmax (optional): device word that receives the float bits of max |out| (activation scale of the tensor-core NC)
int launch_mutual_matching(const float* x, int nA, int nB, float* rowmax, unsigned int* colmax, float* out,
                           unsigned int* absmax, cudaStream_t st);
// second half only: rowmax / colmax were produced by another kernel (nc_combine_kernel)
int launch_mutual_apply(const float* x, int nA, int nB, const float* rowmax, const unsigned int* colmax, float* out,
                        unsigned int* absmax, cudaStream_t st);
int launch_neigh_consensus(const float* x, int hA, int wA, int hB, int wB, const float* w1p, const float* b1p,
                           const float* w2p, float b2, float* hidden, float* out, cudaStream_t st);
int launch_proposals(const float* corr, const uint8_t* code, int hA, int wA, int hB, int wB, int ksize, int upsample,
                     int center, int do_softmax, long long* matches, float* scores, cudaStream_t st);
size_t unique_rows_scratch_bytes(int n);
size_t unique_rank_scratch_bytes();     // zero-initialised, handle-owned scratch of the rank-sort path (n <= 8192)
int launch_unique_rows(const long long* rows, int n, int mutual, const float* scores, float thres, int* ids_out,
                       int* count_out, unsigned char* gscratch, int* rank_scratch, cudaStream_t st);
int launch_select_anchor(const long long* rows, const float* scores, const int* ids, const int* sel, int m, int panc,
                         int pshift, long long* matches_out, float* scores_out, long long* anchors_out, cudaStream_t st);

// ---- topk.cu: corr_to_matches_topk ------------------------------------------------------------------------
constexpr int kTopkMaxSlice = 32768;    // longest slice (cells matched against one cell) the top-k kernel stages
// corr [b][hA*wA][hB*wB]; code NULL or [b][hA*wA][hB*wB] (ks 2..3); outputs [b][k * slices] in the reference's order
int launch_corr_topk(const float* corr, const uint8_t* code, int b, int hA, int wA, int hB, int wB, int k, int ks,
                     int do_softmax, int invert, long long* jA, long long* iA, long long* jB, long long* iB,
                     float* score, cudaStream_t st);

// ---- nc_umma.cu: NeighConsensus on the tensor cores -------------------------------------------------------
struct NcUmmaWeights {
  char* blob = nullptr;           // one allocation backing the two operand images
  __half* img1 = nullptr;         // layer 1 weights, laid out exactly as in shared memory
  __half* img2 = nullptr;         // layer 2 weights
  float wsum1 = 0.f, b1max = 0.f; // bound of the hidden activations: b1max + wsum1 * max|x|
  float inv_sw1 = 1.f, inv_sw2 = 1.f;
};
int nc_umma_pack(const float* w1p, const float* b1p, const float* w2p, NcUmmaWeights& W);
size_t nc_umma_scratch_bytes(size_t V);
size_t nc_umma_xp_bytes(int hA, int wA, int hB, int wB);
int launch_absmax(const float* x, size_t n, unsigned int* out, cudaStream_t st);
int launch_neigh_consensus_umma(const float* x, int hA, int wA, int hB, int wB, const NcUmmaWeights& W, const float* b1p,
                                float b2, const unsigned int* xmax, uint32_t* xp, __half* hidden, float* partial,
                                float* out, float* rowmax, unsigned int* colmax, int l2_mode, int num_sms, cudaStream_t st);

// ---- nc_stack.cu: general NeighConsensus stack (NCNet ImMatchNet) on the tensor cores -----------------------
constexpr int kNcStackMaxLayers = 16;
struct NcStackWeights {
  char* blob = nullptr;           // one allocation backing everything below
  int n_layers = 0, symmetric = 1;
  int ks[kNcStackMaxLayers] = {}, chans[kNcStackMaxLayers] = {};
  float inv_sw[kNcStackMaxLayers] = {};           // 1 / power-of-two weight scale per layer
  const __half* img[kNcStackMaxLayers] = {};     // per layer [k^2][k][k][32][64] swizzled operand images
  const float* bias[kNcStackMaxLayers] = {};     // per layer [16], zero past the layer's channels
  const float* bnd = nullptr;                     // [layers][2][16]: per channel sum |w| (x 1.0001), |b|
};
// weights[l]: HOST fp32 in the reference layout [k][Cout][Cin][k][k][k]; biases[l] [Cout].  Replaces S on success.
int nc_stack_pack(int n_layers, const int* ks, const int* chans, const float* const* weights, const float* const* biases,
                  int symmetric, NcStackWeights& S);
void nc_stack_release(NcStackWeights& S);
size_t nc_stack_scratch_bytes(size_t V);
// x [hA*wA][hB*wB] -> out; xmax: device word holding the float bits of max |x|; scratch: nc_stack_scratch_bytes(V)
int launch_nc_stack(const float* x, int hA, int wA, int hB, int wB, const NcStackWeights& W, const unsigned int* xmax,
                    __half* scratch, float* out, int num_sms, cudaStream_t st);

// ---- preprocess.cu: PIL-exact bicubic resize + ToTensor + Normalize (utils/datasets/preprocess.py:32-60) ----
struct PreprocessCoefs {
  int ho = 0, wo = 0, ht = 0, wt = 0, ksx = 0, ksy = 0;
  size_t o_bx = 0, o_kx = 0, o_by = 0, o_ky = 0;
  int* d = nullptr;               // device: [bounds x][coefs x][bounds y][coefs y]
};
int preprocess_build_coefs(int ho, int wo, int ht, int wt, PreprocessCoefs& C);
int launch_preprocess(const uint8_t* rgb, const PreprocessCoefs& C, const float mean[3], const float stdv[3], float* out,
                      uint8_t* resized_u8, float* gray, uint8_t* tmp, cudaStream_t st);

// ---- refine.cu ---------------------------------------------------------------------------------
// Activation scale applied before the fp16 hi/lo split of the L2-normalised patch features.
constexpr float kActScale = 4096.f;
constexpr int kPatchPos = 256;    // 4 parity planes x 8 x 8 window positions
constexpr int kMainCh = 512;      // (64 + 64 + 128) x 2 images
constexpr int kRgbK = 64;         // 9 taps x 2 images x 3 channels = 54, padded to 64
constexpr int kConv1Steps = 73;   // 9 taps x 8 chunks + 1 rgb chunk (K = 73*64 = 4672)
constexpr int kConv2Steps = 72;   // 9 taps x 8 chunks          (K = 4608)

struct PairFeatures {             // per image: channels-last copies + squared-norm maps
  const float* img;               // [3][H][W]   (level 0 stays NCHW)
  float* nhwc[3];                 // levels 1..3: [h][w][C], C = 64, 64, 128
  __half* nhwc16[3];              // same, fp16, each pixel divided by its own level norm sqrt(nsq[l+1])
  float* nsq[4];                  // levels 0..3: [h][w]
  int H, W;                       // level l is stored at (H >> l) x (W >> l), the index range the reference reads
  // full-resolution window map (fuse_gather = 3): every pixel's patch-normalised 256-channel vector, replicate-padded by
  // kMapPad pixels, [H + 2 pad][map_pitch(W)][256] fp16; rgbn: the normalised rgb triple [..][4] fp16
  __half* wmap;
  __half* rgbn;
};
constexpr int kMapPad = 16;
// Row pitch (pixels) of the window maps: W + 2 pad rounded up to 8, so that every 8-pixel run of the map kernel stays
// in one row whatever W is.  The columns past W + 2 pad are never read.
__host__ __device__ constexpr int map_pitch(int W) { return (W + 2 * kMapPad + 7) & ~7; }
int launch_window_map(const PairFeatures pf[2], cudaStream_t st);

int launch_feature_prep_pair(const float* const feats1[4], const float* const feats2[4], const int H[2], const int W[2],
                             PairFeatures out[2], int fmt, cudaStream_t st);
// rowmap/d_count (optional, device): process only rows rowmap[0..*d_count) (patch slot b <- row rowmap[b]).
int launch_patch_gather(const PairFeatures& f1, const PairFeatures& f2, const void* matches, int is_float, int N,
                        __half* p_hi, __half* p_lo, __half* rgb_hi, __half* rgb_lo, const int* rowmap,
                        const int* d_count, cudaStream_t st);
// Rows whose refined coordinates sit within `tau` px of an integer (and whose offset is not the exact
// relu-clamped -8) are collected, in ascending order, into rowmap / d_count.
int launch_flag_risky(const void* matches_in, int is_float, const float* raw, int N, float tau, float eps_o, int W1,
                      int H1, int W2, int H2, int* rowmap, int* d_count, unsigned long long* totals, cudaStream_t st);

struct FcWeights {                // BN folded, transposed to [in][out] for coalesced reads
  float *w1t, *b1, *w2t, *b2, *w3t, *b3;
};
int launch_fc_parse(const float* pooled, const FcWeights& fc, const void* matches_in, int is_float, int N, int W1,
                    int H1, int W2, int H2, float* matches_out, float* probs_out, float* raw_out, const int* rowmap,
                    const int* d_count, cudaStream_t st);

int launch_finalize_matches(const float* fine, const float* scores, const long long* coarse, int N, float io_thres,
                            const double up[4], double* packed, cudaStream_t st);

// ---- batches of pairs (verify.cu, degensac.cu, pose.cu) -------------------------------------------------------------
// Pair p of a launch reads rows offsets[p] .. offsets[p+1]-1 of `rows` (fp64 (x1, y1, x2, y2) at `stride` doubles
// apart); offsets == nullptr: one pair of n1 rows.  n_dev (device, nullable): pair p uses min(n_p, n_dev[p]) rows.
// Per-row scratch (fp32 rows, pose codes) of a launch is indexed by row - base, base = offsets[0].  Masks are indexed
// by row.  pairs <= kMaxGridY; a batch beyond kBatchScratchBudget bytes of per-pair scratch runs in chunks.
struct PairBatch {
  const double* rows;
  int stride;
  const long long* offsets;
  int n1;
  const double* n_dev;
  long long base;
  long long total;                  // rows of the launch: offsets[pairs] - offsets[0], or n1
  int pairs;
};
inline PairBatch single_pair(const double* rows, int stride, int n, const double* n_dev) {
  return PairBatch{rows, stride, nullptr, n, n_dev, 0, n, 1};
}
constexpr int kMaxGridY = 65535;
constexpr size_t kBatchScratchBudget = (size_t)256 << 20;

// ---- verify.cu: RANSAC for F (model 0, 7-point) / H (model 1, 4-point DLT) / F with DEGENSAC (model 2) and the
// Sampson distance ----------------------------------------------------------------------------------------------------
// rows: fp64 (x1, y1, x2, y2) at `stride` doubles apart; n_dev (optional, device): effective row count min(n, *n_dev).
// Pair p writes model_out[9 p ..], count_out[p] and mask_out[row] for its rows.
size_t verify_scratch_bytes(int pairs, long long rows, bool rounds);
int verify_chunk_pairs();   // pairs per launch within kBatchScratchBudget
int launch_find_model(int model, const PairBatch& B, double px_th, double conf, int max_iters, unsigned long long seed,
                      void* scratch, double* model_out, uint8_t* mask_out, int* count_out, cudaStream_t st);
// Hypotheses 0 .. count-1 without selection: models_out [count*slots][9], counts_out [count*slots] (-1: no model).
int launch_test_hypotheses(int model, const double* rows, int stride, int n, double px_th, unsigned long long seed,
                           int count, void* scratch, double* models_out, int* counts_out, cudaStream_t st);
int launch_sampson_distance(const double* rows, int stride, int n, const double* F, double* out, cudaStream_t st);
// ---- eval.cu: histograms of the Sampson distance against F (passed by value): coarse (columns coarse_col..,
// skipped when < 0), refined (columns 0..3) and refined under mask (nullable); counts_out [3][n_edges], entry
// n_edges-1 = rows considered.
constexpr int kMaxHistEdges = 16;
constexpr int kHistThreads = 1024;
struct EpiHistArgs {
  double F[9];
  double edges[kMaxHistEdges];   // finite, strictly increasing
  int n_edges;                   // 2 .. kMaxHistEdges
};
int launch_epipolar_histograms(const double* rows, int stride, int n, const double* n_dev, int coarse_col,
                               const uint8_t* mask, const EpiHistArgs& a, int* counts_out, cudaStream_t st);
// ---- hpatches.cu: HPatches statistics against a ground-truth H (passed by value): counts_out [n_thr + 1] = rows
// with reprojection error d <= thr[j], then the rows considered; corner_err_out [1] = mean corner distance of H and the
// model of a find_model output buffer H_pred (model at doubles 0..8, int32 count at byte 72), +inf when there is none.
constexpr int kMaxHomThresholds = 16;
struct HomErrArgs {
  double H[9];
  double thr[kMaxHomThresholds];   // finite, > 0, strictly increasing; NaN from n_thr on (no row passes those)
  int n_thr;                       // 1 .. kMaxHomThresholds
  int width, height;               // image 1's size, for the corners
};
int launch_homography_errors(const double* rows, int stride, int n, const double* n_dev, const HomErrArgs& a,
                             const double* H_pred, int* counts_out, double* corner_err_out, cudaStream_t st);
// ---- overlap.cu: cal_overlap_scores' matrix.  ids: flat point3D_ids, image i at offsets[i] .. offsets[i+1]-1 (device);
// bits [n][words] and counts [n] are written by the pack kernel, scores [n][n] (every entry) by the count kernel.
constexpr int kMaxOverlapImages = 1 << 20;
constexpr long long kMaxOverlapPoints = (1LL << 31) - 1;
int launch_overlap_scores(const long long* ids, const long long* offsets, int n, int words, unsigned* bits,
                          int* counts, double* scores, cudaStream_t st);
// ---- degensac.cu: model 2 of launch_find_model (same scratch) and its test hook
int launch_find_model_degensac(const PairBatch& B, double px_th, double conf, int max_iters, unsigned long long seed,
                               void* scratch, double* model_out, uint8_t* mask_out, int* count_out, cudaStream_t st);
// DEGENSAC's degeneracy test of every slot of F hypotheses 0 .. count-1: tri_out [count*3] (-2: no model, -1: not
// degenerate, else the first degenerate triplet), H_out [count*3][9] (its induced H in pixels, zeros otherwise).
size_t verify_degeneracy_scratch_bytes(int n, int count);
int launch_test_degeneracy(const double* rows, int stride, int n, double px_th, unsigned long long seed, int count,
                           void* scratch, int* tri_out, double* H_out, cudaStream_t st);

// ---- pose.cu: essential-matrix RANSAC (5-point) and pose recovery ------------------------------------------------
struct Intrinsics { double fx1, fy1, cx1, cy1, fx2, fy2, cx2, cy2; };   // pixels -> camera coordinates of both views
// Batches as launch_find_model.  intr: DEVICE double [pairs][8] (fx1, fy1, cx1, cy1, fx2, fy2, cx2, cy2), or nullptr:
// K1 for the single pair.  px_th_dev: DEVICE double [pairs], pair p's px_th, or nullptr: px_th for every pair.
size_t essential_scratch_bytes(int pairs, long long rows, bool rounds);
size_t pose_scratch_bytes(int pairs, long long rows);
int essential_chunk_pairs();
int pose_chunk_pairs();
int launch_find_essential(const PairBatch& B, const double* intr, const Intrinsics& K1, double px_th,
                          const double* px_th_dev, double conf, int max_iters, unsigned long long seed, void* scratch,
                          double* E_out, uint8_t* mask_out, int* count_out, cudaStream_t st);
// Hypotheses 0 .. count-1 without selection: models_out [count*10][9], counts_out [count*10] (-1: no model).
int launch_test_essential_hypotheses(const double* rows, int stride, int n, const Intrinsics& K, double px_th,
                                     unsigned long long seed, int count, void* scratch, double* models_out,
                                     int* counts_out, cudaStream_t st);
// E [pairs][9], mask_in / mask_out indexed by row, Rt_out [pairs][12], count_out [pairs].
int launch_recover_pose(const PairBatch& B, const double* intr, const Intrinsics& K1, const double* E,
                        const uint8_t* mask_in, double dist_th, void* scratch, double* Rt_out, uint8_t* mask_out,
                        int* count_out, cudaStream_t st);
// ---- abspose.cu: absolute-pose RANSAC (P3P, Gauss-Newton LO) and the scan lift -------------------------------------
// Rows (u, v, X, Y, Z) in columns 0..4, batches as launch_find_model (a pair is a query).  intr: DEVICE double
// [queries][4] (fx, fy, cx, cy); px_th_dev: DEVICE double [queries] or nullptr (px_th for every query).  Rt_out
// [queries][12] (R row-major, t; x_cam = R X + t), mask_out indexed by row, count_out [queries].
size_t abspose_scratch_bytes(int queries, long long rows, bool rounds);
int abspose_chunk_queries();
int launch_find_absolute_pose(const PairBatch& B, const double* intr, double px_th, const double* px_th_dev,
                              double conf, int max_iters, unsigned long long seed, void* scratch, double* Rt_out,
                              uint8_t* mask_out, int* count_out, cudaStream_t st);
// Hypotheses 0 .. count-1 of one query without selection: intr HOST double [4]; models_out [count*4][12] (centred
// frame), counts_out [count*4] (-1: no pose).
int launch_test_absolute_pose_hypotheses(const double* rows, int stride, int n, const double* intr, double px_th,
                                         unsigned long long seed, int count, void* scratch, double* models_out,
                                         int* counts_out, cudaStream_t st);
// align: HOST double [12], the top 3x4 of the cutout's alignment, row-major.
int launch_lift_scan(const double* scan, int H, int W, const double* align, const double* matches, int match_stride,
                     int n, const double* n_dev, double* rows_out, int row_stride, long long cap, double* count_dev,
                     cudaStream_t st);
// ---- sfm.cu: keypoints, tracks and triangulation against known poses, query 2D-3D rows (semantics in
// include/p2p_b200.h, p2p_sfm_*).  Scratch comes from `ar` (reserved here, which resets it).
constexpr int kMaxSfmTrackPoints = 8;   // points (and rounds) per track
int launch_sfm_keypoints(Arena& ar, const double* m4, long long M, const long long* offsets, int P,
                         const int* pair_img, int both, double px, double* kp_xy, unsigned long long* kp_key,
                         int* kp_of_ep, long long* counts, cudaStream_t st);
int launch_sfm_undistort(const double* xy, const unsigned long long* key, long long cap, const long long* n_dev,
                         const int* img_cam, const double* cams, double* out, cudaStream_t st);
// Synchronises once (the hooking convergence check) and copies counts_dev [6] to counts_host.
int launch_sfm_tracks(Arena& ar, const int* kp_of_ep, long long M, const long long* offsets, int P, const double* E,
                      const double* thr, const double* kp_n, long long n_kp, int* labels, int* obs_kp, int* start,
                      int* tlen, long long* counts_dev, long long* counts_host, cudaStream_t st);
int launch_sfm_triangulate(Arena& ar, const int* obs_kp, const int* start, const int* tlen, int n_tracks,
                           long long n_kp, const double* kp_xy, const double* kp_n, const unsigned long long* kp_key,
                           const double* img, const int* img_cam, const double* cams, double reproj_px,
                           double cos_min, double* pts, int* pt_len, double* pt_err, int* kp_point, long long* counts,
                           cudaStream_t st);
int launch_sfm_query_rows(Arena& ar, const double* m4, long long M, const long long* offsets, int P,
                          const int* pair_img, int n_queries, double px, const int* qkp_of_ep,
                          const unsigned long long* qkp_key, const double* qkp_n, const double* q_intr,
                          const unsigned long long* kp_key, const double* kp_xy, const int* kp_point, long long n_kp,
                          const double* pts, double* rows, long long* q_offsets, cudaStream_t st);
// ---- keypoints.cu: SuperPoint's keypoints and descriptors, exact nearest-neighbour matching (semantics in
// include/p2p_b200.h, p2p_sp_* and p2p_match_descriptors_batch).  Scratch comes from `ar` (reserved here).
constexpr int kSpMaxNmsRadius = 16;
constexpr int kSpMaxDescDim = 512;      // descriptor channels the sampling kernel holds per warp
constexpr int kMatchMaxDim = 1024;
int launch_sp_keypoints(Arena& ar, const float* logits, int B, int Hc, int Wc, int r, float thr, int border, int k,
                        float* smap_out, float* kp, float* kp_score, long long* counts, cudaStream_t st);
int launch_sp_descriptors(Arena& ar, const float* raw, int B, int D, int Hc, int Wc, const float* kp,
                          const long long* kp_off, long long N, float* out, cudaStream_t st);
int launch_match_descriptors(Arena& ar, const float* d0, const float* d1, const long long* off0,
                             const long long* off1, int K, int D, int max_n0, int max_n1, long long n0, long long n1,
                             int mutual, int has_min, double min_sim, int has_ratio, double ratio, int impl,
                             int* match, double* sim, double* tc_sim, int* tc_idx, double* eps_out,
                             int* n_fixed, cudaStream_t st);
// ---- superglue.cu: SuperGlue's log-domain Sinkhorn and mutual match extraction in one cooperative launch (semantics
// in include/p2p_b200.h, p2p_sg_sinkhorn).  Scratch (a transposed copy of the scores, u, v and the argmaxes) comes from
// `ar` (reserved here); `sms` caps the persistent grid at that many SMs' worth of co-resident blocks.
constexpr int kSgMaxPoints = 1 << 20;
constexpr int kSgMaxIters = 100000;
int launch_sg_sinkhorn(Arena& ar, const float* scores, int B, int n, int m, const float* alpha, int iters, float thr,
                       float* log_assign, int* matches0, int* matches1, float* mscores0, float* mscores1, int sms,
                       cudaStream_t st);
// ---- relpose.cu: relative-pose statistics of a batch (one block per pair, pairs = B.pairs, any count): pair p writes
// out[p * out_stride ..] = cos of the rotation and translation-direction errors of Rt_est [p] against Rt_gt [p]
// (NaN when n_inliers[p] <= 0), then int32 [n_thr + 1]: rows with symmetric epipolar error < thr[j], rows considered.
constexpr int kMaxRelposeThresholds = 16;
struct RelposeErrArgs {
  double thr[kMaxRelposeThresholds];   // finite, > 0, strictly increasing; NaN from n_thr on (no row passes those)
  int n_thr;                           // 1 .. kMaxRelposeThresholds
};
int launch_relpose_errors(const PairBatch& B, const double* intr, const double* Rt_gt, const double* Rt_est,
                          const int* n_inliers, const RelposeErrArgs& a, double* out, int out_stride, cudaStream_t st);

// Tensor-core FC path helpers: pooled fp32 -> fp16 hi/lo A operand (times `scale`); final Linear(256,5) +
// parse_regressor_out of h2 = (h2_hi + h2_lo) * inv_scale.
int launch_pooled_split(const float* pooled, int n, float scale, __half* hi, __half* lo, const int* d_count, cudaStream_t st);
int launch_fc3_parse(const __half* h2_hi, const __half* h2_lo, float inv_scale, const float* w3t, const float* b3, const void* matches_in,
                     int is_float, int N, int W1, int H1, int W2, int H2, float* matches_out, float* probs_out,
                     float* raw_out, const int* rowmap, const int* d_count, cudaStream_t st);

// One k-step of an implicit GEMM: where the [128 rows x 64 ch] A box starts and which K offset of
// the K-major weight matrix it multiplies.
struct KStep {
  short c0;                       // channel coordinate of the A box
  signed char x, y;               // spatial start (may be -1: TMA zero-fills out-of-bounds)
  signed char plane;              // parity plane (conv1) or 0
  signed char kind;               // 0 = main activation tensor, 1 = rgb im2col tensor
  short pad;
  int bk;                         // K coordinate in the weight matrix
};

// CUDA-core debug GEMM over exactly the tensors the wgmma kernel consumes (bring-up checker;
// not a product path: selected only by p2p_set_option("gemm_impl", 1)).
struct GemmOperands {
  const __half *a_hi, *a_lo;      // main A tensor [N][planes][8][8][512]
  const __half *r_hi, *r_lo;      // rgb A tensor  [N][64][64]  (nullptr for conv2)
  const __half *b_hi, *b_lo;      // weights [512][Ktot], K-major
  int planes;                     // 4 (conv1) or 1 (conv2)
  int ktot;                       // K extent of B
  int n_patches;
  int passes;                     // 1: hi*hi ; 3: hi*hi + lo*hi + hi*lo
  const KStep* steps;             // device array
  int nsteps;
};
struct ConvEpilogue {
  const float* scale;             // [512] = 1 / (act_scale * w_scale[o])
  const float* bias;              // [512]
  int mode;                       // 0: write y1 hi/lo (scaled by y_scale); 1: relu + 8x8 max -> pooled
  float y_scale;
  __half *y_hi, *y_lo;            // [N][8][8][512]
  float* pooled;                  // [N][512]
};
int launch_conv_gemm_simt(const GemmOperands& g, const ConvEpilogue& e, cudaStream_t st);

}  // namespace p2p
