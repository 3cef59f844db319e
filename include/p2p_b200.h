/* libp2p_b200.so -- C ABI of the H100-native (sm_90a) Patch2Pix correlate-and-refine path.
 *
 * The reference (GrumpyZhou/patch2pix) has no FFI / operator registry: its boundary for this path
 * is the Python method surface of `networks.patch2pix.Patch2Pix` (SURVEY.md s8b).  Each entry point
 * below therefore cites the reference method / function (file:line in the reference repo) whose
 * computation it replaces; `patch2pix_b200/model.py` binds them through ctypes behind the same
 * method names, and INTEGRATION.md shows the stub a maintainer would add to the reference.
 *
 * Conventions: every function returns 0 on success, a negative code on failure
 * (-1 invalid argument, -2 CUDA/driver error, -3 out of memory) and never throws;
 * `p2p_last_error()` returns a thread-local description of the last failure.
 * All data pointers are DEVICE pointers to caller-owned, contiguous memory on the handle's
 * device unless marked HOST.  Work is enqueued on `stream` (a cudaStream_t passed as void*);
 * no entry point synchronises the device.  The library owns only packed weights and scratch,
 * both freed by `p2p_destroy`.  There is no CPU fallback: shape violations are errors.
 */
#ifndef P2P_B200_H_
#define P2P_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define P2P_API __attribute__((visibility("default")))

typedef struct p2p_handle_s* p2p_handle_t;

/* HOST pointers to fp32 arrays laid out exactly as in the reference `state_dict`
 * (networks/modules.py:76-99): conv.0.weight [512,518,3,3]; conv.1.{weight,bias,running_mean,
 * running_var} [512]; conv.2.weight [512,512,3,3]; conv.3.* [512]; fc.0.weight [512,512],
 * fc.0.bias; fc.1.* [512]; fc.3.weight [256,512], fc.3.bias; fc.4.* [256]; fc.6.weight [5,256],
 * fc.6.bias [5].  BatchNorm is folded (eval mode, eps) while packing. */
typedef struct p2p_bn_s {
  const float* weight;
  const float* bias;
  const float* running_mean;
  const float* running_var;
} p2p_bn_t;

typedef struct p2p_regressor_weights_s {
  const float* conv0_weight;
  p2p_bn_t conv1_bn;
  const float* conv2_weight;
  p2p_bn_t conv3_bn;
  const float* fc0_weight;
  const float* fc0_bias;
  p2p_bn_t fc1_bn;
  const float* fc3_weight;
  const float* fc3_bias;
  p2p_bn_t fc4_bn;
  const float* fc6_weight;
  const float* fc6_bias;
  float bn_eps;
} p2p_regressor_weights_t;

P2P_API const char* p2p_last_error(void);
P2P_API int p2p_version(void);

/* One handle per device; not thread-safe; replaces the module state built by
 * Patch2Pix.__init__ (networks/patch2pix.py:13-61) for the hot path. */
P2P_API int p2p_create(int device, p2p_handle_t* out);
P2P_API int p2p_destroy(p2p_handle_t h);

/* NeighConsensus parameters, HOST fp32, reference layout (networks/ncn/conv4d.py:118-120):
 * w1 = ncn.conv.0.weight [3,16,1,3,3,3], b1 [16], w2 = ncn.conv.2.weight [3,1,16,3,3,3], b2 [1]. */
P2P_API int p2p_set_ncn_weights(p2p_handle_t h, const float* w1, const float* b1, const float* w2, const float* b2);

/* A general NeighConsensus stack (NCNet's ImMatchNet, networks/ncn/model.py:124-155), packed beside the Patch2Pix weights
 * above: n_layers Conv4d layers (1..16), kernel_sizes[l] in {3, 5}, channels[l] in 1..16 with channels[n_layers-1] == 1.
 * weights[l]: HOST fp32 in the reference's pre-permuted layout [k, Cout, Cin, k, k, k] (conv4d.py:118-120), Cin = 1 for
 * layer 0 and channels[l-1] after; biases[l] [Cout].  symmetric != 0: conv(x) + conv(x^T)^T (symmetric_mode). */
P2P_API int p2p_set_nc_stack_weights(p2p_handle_t h, int n_layers, const int* kernel_sizes, const int* channels,
                                     const float* const* weights, const float* const* biases, int symmetric);

/* which: 0 = regress_mid, 1 = regress_fine (networks/patch2pix.py:53-58). */
P2P_API int p2p_set_regressor_weights(p2p_handle_t h, int which, const p2p_regressor_weights_t* w);

/* Options: "mid_passes"/"fine_passes" (1 = fp16 operands, 3 = fp16 hi/lo split, fp32-grade),
 * "corr_passes" (0 = CUDA-core fp32 correlation, 1/3 = tensor-core), "seg_len" (k-steps per
 * tensor-core accumulation segment, 0 = whole K), "gemm_impl" (0 = wgmma, 1 = CUDA-core checker),
 * "num_sms" (persistent grid size, 0 = all), "profile" (1 = record per-kernel CUDA events),
 * "mid_band" (thousandths of a pixel, default 26 = 2x the largest 1-pass/3-pass difference measured over 125k DISTINCT
 * coordinates; with mid_passes = 3 every row is first computed 1-pass and
 * only rows with a coordinate within the band of an integer -- where trunc(mid) could differ from the
 * reference -- are re-computed 3-pass; 0 = 3-pass for every row), "fuse_gather" (conv1 A operand of the 1-pass launches; default 3 = per-image window map + strided TMA boxes, no
 * producer warps; 1 = gathered in producer warps; 2 = first-generation fused kernel; 0 = separate gather kernel + TMA
 * of a materialised patch tensor; all four give bit-identical results except 0, which skips one fp16 rounding),
 * "nc_impl" (default 1: NeighConsensus on the tensor cores, nc_umma.cu; 0: fp32 CUDA-core kernels, B grid <= 3072 cells),
 * "nc_l2_mode" (layout of NC layer 2's block of hidden lines: 0 = chosen per shape, 1 = one haloed block per tile,
 * 2 = one block per column tap; bit-identical results), "unique_impl" (default 1: rank sort over the whole GPU for lists of
 * up to 8192 rows; 0: single-block bitonic network; identical results), "fc_impl" (default 1: the 512-512 and 512-256 Linear layers run on
 * the tensor cores, 3-pass; 0: fp32 CUDA-core FC kernel), "share_windows" (default 1: in the mid stage's window-map
 * 1-pass conv1, a half-group of 4 rows (rows 8g..8g+3 on image 2, 8g+4..8g+7 on image 1) with equal window origins
 * computes that image's half of conv1 once; shared rows differ from 0 by one reordering of an fp32 sum, all other rows
 * are bit-identical; 0: every row's whole conv1), "epi_async" (default 1: the 256-wide 1-pass conv1 / conv2 launches
 * take their epilogue straight from the wgmma fragments, conv1's fp16 output leaving by TMA store; 0: through the fp32
 * shared-memory staging buffer; bit-identical results), "tile_trace" (default 0; 1: the conv GEMM launches and
 * p2p_test_gemm record a per-tile phase trace, read with p2p_tile_trace_read; setting it clears the trace).
 * p2p_get_option also reads "shared_rows": the rows that shared a window half in the last mid-stage call
 * (synchronises), "frag_epi_launches": conv launches run with the fragment epilogues so far, and "tile_traces": the
 * traced launches since tile_trace was set. */
P2P_API int p2p_set_option(p2p_handle_t h, const char* key, int value);
P2P_API int p2p_get_option(p2p_handle_t h, const char* key, int* value);
/* Number of kernel launches enqueued by this handle since creation (bench.py's gpu_launches). */
P2P_API int p2p_launch_count(p2p_handle_t h, long long* count);

/* Per-kernel-group device times (CUDA events on the launching stream), accumulated while the
 * "profile" option is 1.  Synchronises on the recorded events, returns ms and launch-group counts
 * per kind, and clears the log. */
enum {
  P2P_PROF_L2NORM = 0, P2P_PROF_CORR = 1, P2P_PROF_MUTUAL = 2, P2P_PROF_NC = 3, P2P_PROF_PROPOSALS = 4,
  P2P_PROF_PREP = 5, P2P_PROF_GATHER_MID = 6, P2P_PROF_CONV1_MID = 7, P2P_PROF_CONV2_MID = 8, P2P_PROF_FC_MID = 9,
  P2P_PROF_GATHER_FINE = 10, P2P_PROF_CONV1_FINE = 11, P2P_PROF_CONV2_FINE = 12, P2P_PROF_FC_FINE = 13,
  P2P_PROF_GATHER_BAND = 14, P2P_PROF_CONV1_BAND = 15, P2P_PROF_CONV2_BAND = 16, P2P_PROF_FC_BAND = 17,
  P2P_PROF_FLAG = 18, P2P_PROF_KINDS = 19
};
P2P_API int p2p_profile_read(p2p_handle_t h, float* ms_by_kind, int* count_by_kind, int nkinds);

/* ---- coarse stage: Patch2Pix.forward_coarse_match (networks/patch2pix.py:120-136) -------------
 * feat1 [c,h1,w1], feat2 [c,h2,w2] fp32 (one batch item).  ksize 1 or 2.
 * corr4d_out [hp1*wp1, hp2*wp2] fp32 with hp = h/ksize (the final MutualMatching output).
 * delta_code_out (ksize 2 only, may be NULL for ksize 1): uint8 [hp1*wp1, hp2*wp2],
 * code = ((di*k+dj)*k+dk)*k+dl of maxpool4d (networks/modules.py:11-34).
 * Optional stage taps for parity tests (may be NULL): pooled_out (after maxpool4d),
 * ncn_out (after NeighConsensus, before the second MutualMatching). */
P2P_API int p2p_coarse(p2p_handle_t h, const float* feat1, const float* feat2, int c, int h1, int w1, int h2, int w2,
               int ksize, float* corr4d_out, uint8_t* delta_code_out, float* pooled_out, float* ncn_out,
               void* stream);

/* Same, for a channels-last fp16 layer-3 map: feat1 [h1][w1][c], feat2 [h2][w2][c] (what an fp16 / channels_last
 * backbone emits; the L2-normalise + K-major re-layout pass then needs no transpose).  Identical arithmetic from there on. */
P2P_API int p2p_coarse_nhwc16(p2p_handle_t h, const void* feat1_nhwc16, const void* feat2_nhwc16, int c, int h1, int w1, int h2,
               int w2, int ksize, float* corr4d_out, uint8_t* delta_code_out, float* pooled_out, float* ncn_out,
               void* stream);

/* maxpool4d's four int64 delta tensors (max_i,max_j,max_k,max_l) from the packed code. */
P2P_API int p2p_delta_unpack(p2p_handle_t h, const uint8_t* code, long long n, int ksize, int64_t* di, int64_t* dj,
                     int64_t* dk, int64_t* dl, void* stream);
/* Inverse, for callers that hand in reference-style delta4d tensors. */
P2P_API int p2p_delta_pack(p2p_handle_t h, const int64_t* di, const int64_t* dj, const int64_t* dk, const int64_t* dl,
                   long long n, int ksize, uint8_t* code, void* stream);

/* MutualMatching alone (networks/ncn/model.py:157-176) on [nA, nB]. */
P2P_API int p2p_mutual_matching(p2p_handle_t h, const float* in, int nA, int nB, float* out, void* stream);
/* NeighConsensus alone (networks/ncn/model.py:145-155) on [hA,wA,hB,wB] (timed as P2P_PROF_NC). */
P2P_API int p2p_neigh_consensus(p2p_handle_t h, const float* in, int hA, int wA, int hB, int wB, float* out, void* stream);
/* The stack of p2p_set_nc_stack_weights alone on [hA,wA,hB,wB] fp32 (tensor cores; timed as P2P_PROF_NC). */
P2P_API int p2p_nc_stack(p2p_handle_t h, const float* in, int hA, int wA, int hB, int wB, float* out, void* stream);
/* ImMatchNet.forward_feat (networks/ncn/model.py:289-312) for one pair: L2-normalised features feat1 [c,h1,w1],
 * feat2 [c,h2,w2] (c % 64 == 0) -> correlation, maxpool4d (ksize 2) -> MutualMatching -> the stack ->
 * MutualMatching.  corr4d_out and delta_code_out as for p2p_coarse. */
P2P_API int p2p_ncnet_coarse(p2p_handle_t h, const float* feat1, const float* feat2, int c, int h1, int w1, int h2, int w2,
                             int ksize, float* corr4d_out, uint8_t* delta_code_out, void* stream);

/* ---- proposals: Patch2Pix.cal_coarse_matches (networks/patch2pix.py:340-375, sort=False) over
 * corr_to_matches (networks/ncn/extract_ncmatches.py:6-94).  corr4d [hA*wA, hB*wB]; delta_code may be
 * NULL (ksize 1).  matches_out int64 [hB*wB + hA*wA, 4] rows (x1,y1,x2,y2): first the best A cell for
 * every B cell, then the best B cell for every A cell; scores_out fp32 same length. */
P2P_API int p2p_proposals(p2p_handle_t h, const float* corr4d, const uint8_t* delta_code, int hA, int wA, int hB, int wB,
                  int ksize, int upsample, int center, int do_softmax, int64_t* matches_out, float* scores_out,
                  void* stream);

/* ---- top-k matches: corr_to_matches_topk (networks/ncn/extract_ncmatches.py:96-158) for a batch of b volumes in
 * one launch.  corr4d fp32 [b][hA*wA][hB*wB]; delta_code NULL (ksize 1) or uint8 [b][hA*wA][hB*wB] packed as by
 * p2p_delta_pack.  A slice is the cells matched against one cell: forward (invert 0) the hA*wA A cells of each of the
 * N = hB*wB B cells, inverted the hB*wB B cells of each of the N = hA*wA A cells.  Each slice yields its topk best
 * cells, ranked by the raw value, descending; exact ties go to the lowest flat cell index.  Outputs are int64 / fp32
 * [b][topk * N] cell indices (index * ksize + delta with delta_code) and scores (exp(x - max) / sum over the slice,
 * or x for do_softmax 0), rank-major forward (rank r of cell s at r * N + s), cell-major inverted (s * topk + r).
 * Limits: slices of at most 32768 cells, 1 <= topk <= slice length, b <= 65535.  Timed as P2P_PROF_PROPOSALS. */
P2P_API int p2p_proposals_topk(p2p_handle_t h, const float* corr4d, const uint8_t* delta_code, int b, int hA, int wA,
                               int hB, int wB, int topk, int ksize, int do_softmax, int invert, int64_t* jA_out,
                               int64_t* iA_out, int64_t* jB_out, int64_t* iB_out, float* scores_out, void* stream);

/* ---- the np.unique part of filter_coarse (networks/utils.py:38-50): lexicographically sorted
 * first-occurrence indices of the distinct rows (mutual != 0: only rows occurring more than once).
 * rows int64 [n,4] with coordinates in [0,65535], n <= 4 Mi (lists beyond 16384 rows sort in global scratch); ids_out int32 [n]; count_out int32 [4] =
 * {number of ids, 1 if a coordinate was out of range, number of those ids whose score > thres,
 * number of ALL rows whose score > thres}; the last two (scores may be NULL -> 0) let the caller
 * evaluate filter_coarse's score threshold (utils.py:53) without a second device sync. */
P2P_API int p2p_unique_rows(p2p_handle_t h, const int64_t* rows, int n, int mutual, const float* scores, float thres,
                    int32_t* ids_out, int32_t* count_out, void* stream);

/* ---- the index arithmetic that follows np.unique in filter_coarse (networks/utils.py:51-69: matches[ids][ids2],
 * scores likewise) fused with Patch2Pix.shift_to_anchors (networks/patch2pix.py:377-402).
 * Output row r <- rows[ids[sel[r]]] (ids, sel int32 DEVICE, either may be NULL = identity); m output rows.
 * panc 8: anchors_out int64 [m*8,4] = every selected row + the reference's 8-row template
 * ((-p,-p,0,0),(p,-p,0,0),(-p,p,0,0),(p,p,0,0),(0,0,-p,-p),(0,0,p,-p),(0,0,-p,p),(0,0,p,p)); panc 1: anchors_out unused.
 * matches_out int64 [m,4] / scores_out fp32 [m] may be NULL. */
P2P_API int p2p_select_anchor(p2p_handle_t h, const int64_t* rows, const float* scores, const int32_t* ids,
                      const int32_t* sel, int m, int panc, int pshift, int64_t* matches_out, float* scores_out,
                      int64_t* anchors_out, void* stream);

/* ---- refine: Patch2Pix.forward_fine_match for one batch item (networks/patch2pix.py:157-218):
 * select_local_patch_feats + L2 normalise + FeatRegressNet + parse_regressor_out.
 * feats1/feats2: HOST arrays of 4 DEVICE pointers, the ResNet.forward_all levels 0..3 (networks/resnet.py:138-157) as
 * the backbone produces them for an H x W image: image [3,H,W], conv1-relu [64,h1,w1], layer1 [64,h2,w2],
 * layer2 [128,h3,w3] with the ceiling chain h1 = ceil(H/2), h2 = ceil(h1/2), h3 = ceil(h2/2) (same for w).  Any
 * H, W >= 8 is accepted (below 8 the reference's level-3 clamp bound W // 8 - 1 is negative); only the top-left
 * (H >> l) x (W >> l) of level l is read, the index range of the reference's per-level clamp.  For multiples of 8 the
 * chain is H/2, H/4, H/8.
 * `p2p_refine_prepare` must be called once per image pair before p2p_refine (it builds channels-last
 * copies and norm maps); matches_in [n,4] int64 (is_float = 0) or fp32 (is_float = 1);
 * matches_out fp32 [n,4]; probs_out fp32 [n]. */
P2P_API int p2p_refine_prepare(p2p_handle_t h, const float* const* feats1, const float* const* feats2, int H1, int W1,
                       int H2, int W2, void* stream);
/* Same, with levels 1..3 as channels-last fp16 maps [h][w][C] of the same ceiling-chain sizes (level 0, the image,
 * stays [3,H,W] fp32). */
P2P_API int p2p_refine_prepare_nhwc16(p2p_handle_t h, const void* const* feats1, const void* const* feats2, int H1, int W1,
                       int H2, int W2, void* stream);
P2P_API int p2p_refine(p2p_handle_t h, int which, const void* matches_in, int is_float, int n, float* matches_out,
               float* probs_out, void* stream);
/* Test access: copies the intermediate buffers of the handle's last p2p_refine call, as they stand after its last pass,
 * into the caller's DEVICE buffers (each may be NULL).  Valid until the next p2p_refine on the handle; synchronises
 * `stream` after a risk-band call.  info_out HOST int32 [4] = {m: rows of the last pass, passes of the last pass (1 or 3),
 * 1 if the last pass was the risk band's 3-pass subset, 1 if the FC ran on the tensor cores}.  After a risk-band call the
 * buffers hold the band's m flagged rows, slot s holding row rows_out[s] (ascending); otherwise slot s is row s of the n.
 * scales_out HOST float [4]: the power-of-two scales the buffers carry: y_scale, then the FC operand scales of
 * pooled, h1 and h2.  rows_out int32 [m]; y_hi / y_lo fp16 [m][64][512], the conv1 output (BN folded) times y_scale
 * at output pixel y * 8 + x, y_hi + y_lo after a 3-pass pass (y_lo NULL after a 1-pass one); pooled fp32 [m][512]
 * (unscaled); h1_hi / h1_lo fp16 [m][512] and h2_hi / h2_lo fp16 [m][256], the FC hidden layers times their scales
 * (tensor-core FC only); raw_out fp32 [n][5], the regressor outputs of every row (the band's rows from its 3-pass pass). */
P2P_API int p2p_refine_taps(p2p_handle_t h, int32_t* info_out, float* scales_out, int32_t* rows_out, void* y_hi, void* y_lo,
                            float* pooled, void* h1_hi, void* h1_lo, void* h2_hi, void* h2_lo, float* raw_out,
                            void* stream);

/* ---- tail of estimate_matches (utils/eval/model_helper.py:97-109): inlier filter `scores > io_thres` ("keep everything
 * if nothing passes"), row order preserved, and `upscale * matches` in float64, so that ONE device->host copy returns
 * the final result.  fine fp32 [n,4] (NULL for eval_type 'coarse': the refined columns repeat the coarse ones), scores
 * fp32 [n], coarse int64 [n,4], upscale4 HOST double[4] = (sx1, sy1, sx2, sy2).  packed_out DEVICE double [n*9 + 1]:
 * rows (x1,y1,x2,y2 refined, score, x1,y1,x2,y2 coarse), packed_out[n*9] = number of rows kept. */
P2P_API int p2p_finalize_matches(p2p_handle_t h, const float* fine, const float* scores, const int64_t* coarse, int n,
                         float io_thres, const double* upscale4, double* packed_out, void* stream);

/* ---- image preprocessing: the tensor half of load_im_flexible (utils/datasets/preprocess.py:32-60):
 * transforms.functional.resize(img, (ht, wt), Image.BICUBIC) -> ToTensor -> Normalize(ImageNet mean/std) for a decoded
 * 8-bit RGB image.  Pillow's 8-bit resampling (fixed-point, antialiased bicubic, horizontal then vertical pass) is
 * reproduced bit-exactly.  rgb_hwc: DEVICE uint8 [ho][wo][3]; out_chw: DEVICE fp32 [3][ht][wt];
 * resized_hwc_out (optional, may be NULL): DEVICE uint8 [ht][wt][3], the resized image before normalisation.
 * (ht, wt) come from cal_rescale_size (preprocess.py:83-91), computed by the caller. */
P2P_API int p2p_preprocess_image(p2p_handle_t h, const uint8_t* rgb_hwc, int ho, int wo, int ht, int wt, float* out_chw,
                         uint8_t* resized_hwc_out, void* stream);
/* The same for load_im_tensor (utils/datasets/preprocess.py:7-30), the loader of the refiner entry point: (ht, wt) are
 * the caller's int(round(ho * s)), int(round(wo * s)), or (ho, wo) when the image is not downscaled.  gray_hw
 * (optional, may be NULL): DEVICE fp32 [ht][wt], Pillow's convert('L') of the resized 8-bit image
 * ((19595 R + 38470 G + 7471 B + 0x8000) >> 16) divided by 255, written by the same launch as out_chw. */
P2P_API int p2p_preprocess_image_gray(p2p_handle_t h, const uint8_t* rgb_hwc, int ho, int wo, int ht, int wt,
                         float* out_chw, float* gray_hw, void* stream);

/* ---- match verification: what every consumer of the match list does next in the reference -- pydegensac's
 * findFundamentalMatrix / findHomography in examples/visualize_matches.ipynb (first cell), the F / pose RANSAC of
 * utils/train/eval_epoch_immatch.py:51-80 and utils/eval/geometry.py:32-71 -- as RANSAC on the device.
 * rows: fp64 (x1, y1, x2, y2) in pixels, row r at rows + r * row_stride (row_stride >= 4; 9 consumes the packed_out of
 * p2p_finalize_matches in place); n_dev (nullable, DEVICE double): use min(n, *n_dev) rows, e.g. packed_out + n * 9.
 * model 0 = fundamental matrix, x2^T F x1 = 0 (7-point minimal solver, inlier iff the Sampson error
 * dd^2 / (l1x^2 + l1y^2 + l2x^2 + l2y^2) < px_th^2); model 1 = homography x2 ~ H x1 (4-point DLT, inlier iff the
 * one-sided transfer error |pi(H x1) - x2|^2 < px_th^2 with (H x1)_z > 0).  Hartley-normalised minimal samples from a
 * counter-based generator of (seed, hypothesis, draw); rounds of 1024 hypotheses stop, on the device, once
 * log(1 - conf) / log(1 - w^s) hypotheses have been drawn (w the best inlier ratio) or at max_iters; the winner (most
 * inliers, ties to the lowest (hypothesis, root) index) is refitted on its inliers (F: 8-point + rank 2; H: DLT) while
 * the count grows.  Bit-reproducible.  model_out DEVICE double [9] row-major (F: unit Frobenius norm, H: H[2][2] = 1),
 * mask_out DEVICE uint8 [n], n_inliers_out DEVICE int32: 0 = no model (fewer rows than a sample or every sample
 * degenerate; model and mask zeroed), -1 = a coordinate is not finite (model NaN, mask zeroed).
 * model 2 = F with the DEGENSAC plane-degeneracy check (Chum, Werner & Matas, CVPR 2005), pydegensac's
 * findFundamentalMatrix: model 0's rounds, scoring, select, stopping bound, LO and outputs, plus, in each round, an
 * H-degeneracy test of the round's records (every slot whose count beats the best so far and all earlier slots of the
 * round: the models a sequential RANSAC would adopt, the round's winner among them), in slot order.  For each triplet
 * {0,1,2}, {3,4,5}, {0,1,6}, {3,4,6}, {2,5,6} of the record's 7-point sample (hypothesis first + slot / 3) the
 * homography induced by F and the three points (Hartley & Zisserman, result 13.6: H = A - e' (M^-1 b)^T with
 * A = [e']x F, M the rows x_i^T, b_i = (x'_i x A x_i)^T (x'_i x e') / |x'_i x e'|^2) is built in fp64 in the Hartley-
 * normalised coordinates; the sample is degenerate when at least 5 of its 7 points have a one-sided transfer error
 * below h_th = 2 px_th (the notebook's 2 px H threshold beside its 1 px F threshold); a vanishing e', a point at the
 * epipole or collinear x_i give no H.  The first degenerate record starts a plane-and-parallax round: its H is refitted
 * on the rows within h_th (DLT while the count grows, fp64 tests), then 1024 two-row samples from a second stream of
 * the generator (seed ^ 0x5851F42D4C957F2D, hypotheses first .. first + 1023; a draw within h_th of H is re-drawn,
 * at most 64 draws) give e' = (H x_a x x'_a) x (H x_b x x'_b) and F = [e']x H, scored as F and adopted only with
 * strictly more inliers.  One such round finds a pair of off-plane inliers among the H outliers (fraction w) with
 * probability 1 - (1 - w^2)^1024, 0.998 at w = 8 %. */
P2P_API int p2p_find_model(p2p_handle_t h, int model, const double* rows, int row_stride, int n, const double* n_dev,
                   double px_th, double conf, int max_iters, unsigned long long seed, double* model_out, uint8_t* mask_out,
                   int32_t* n_inliers_out, void* stream);
/* The reference's sampson_distance (utils/eval/measure.py:18-40, eps = 1e-8) in fp64: dist_out[r] =
 * (x2^T F x1)^2 / (eps + l1x^2 + l1y^2 + l2x^2 + l2y^2).  F DEVICE double [9], dist_out DEVICE double [n]. */
P2P_API int p2p_sampson_distance(p2p_handle_t h, const double* rows, int row_stride, int n, const double* F,
                         double* dist_out, void* stream);
/* The three Sampson-distance histograms of the reference's validation loop (utils/train/eval_epoch_immatch.py:62-91:
 * cdist, fdist, indist binned as check_inliers_distr does), in one launch and without a host sync.  rows / row_stride /
 * n / n_dev as p2p_find_model: m = min(n, *n_dev) rows, refined (x1, y1, x2, y2) in columns 0..3, the coarse ones in
 * columns coarse_col..coarse_col+3 (-1: no coarse histogram; row_stride 9 with coarse_col 5 reads the packed_out of
 * p2p_finalize_matches in place).  The distance is bit-identical to p2p_sampson_distance.  F HOST double [9] and edges
 * HOST double [n_edges] (2 <= n_edges <= 16, finite, strictly increasing; anything else returns -1) are passed by value
 * to the kernel.  Binning as np.histogram(d, edges): bin i counts edges[i] <= d < edges[i+1], the last bin also
 * d == edges[n_edges-1]; NaN, inf and values outside the edges are not counted.  counts_out DEVICE int32 [3][n_edges]:
 * histogram 0 = coarse over the m rows (all zero when coarse_col = -1), 1 = refined over the m rows, 2 = refined over
 * the rows with mask[r] != 0 (mask DEVICE uint8 [n], nullable: NULL zeroes histogram 2); entries 0 .. n_edges-2 of each
 * are the bin counts and entry n_edges-1 the number of rows considered (the divisor of the reference's ratios, which
 * includes the rows outside the bins).  Integer counts: identical across runs and num_sms settings. */
P2P_API int p2p_epipolar_histograms(p2p_handle_t h, const double* rows, int row_stride, int n, const double* n_dev,
                                    int coarse_col, const double* F, const uint8_t* mask, const double* edges,
                                    int n_edges, int32_t* counts_out, void* stream);
/* The per-pair statistics of the HPatches evaluation (patch2pix_b200/hpatches.py), in one launch and without a host
 * sync.  rows / row_stride / n / n_dev as p2p_find_model: m = min(n, *n_dev) rows (x1, y1, x2, y2) in columns 0..3
 * (row_stride 9 reads the packed_out of p2p_finalize_matches in place).  H_gt HOST double [9] (row-major, image 1 ->
 * image 2) and thresholds HOST double [n_thr] (1 <= n_thr <= 16, finite, > 0, strictly increasing; anything else
 * returns -1) are passed by value to the kernel.  A row's reprojection error is d = |pi(H_gt [x1, y1, 1]^T) - (x2, y2)|
 * in fp64, every product and sum rounded on its own ((h0 x + h1 y) + h2, no fused multiply-add), correctly rounded
 * division and square root; it counts at threshold t iff d <= t, so NaN and inf never count.  counts_out DEVICE int32
 * [n_thr + 1]: the count at each threshold, then m.  H_pred is a DEVICE p2p_find_model output buffer (model at doubles
 * 0..8, int32 inlier count at byte 72).  corner_err_out DEVICE double [1]: the mean over the corners (0, 0),
 * (width-1, 0), (0, height-1), (width-1, height-1) of |pi(H_gt c) - pi(H_pred c)|, summed in that order and divided
 * by 4; +inf when the inlier count is <= 0, when a corner projects with w = 0 under either H, or when the mean is not
 * finite.  Both outputs are written with plain stores (no zeroing needed) and are identical across runs. */
P2P_API int p2p_homography_errors(p2p_handle_t h, const double* rows, int row_stride, int n, const double* n_dev,
                                  const double* H_gt, const double* H_pred, int width, int height,
                                  const double* thresholds, int n_thr, int32_t* counts_out, double* corner_err_out,
                                  void* stream);
/* The image-overlap matrix of the reference's validation-pair precompute (utils/colmap/data_loading.py:54-70,
 * cal_overlap_scores), in two launches and without a host sync.  Image i's keypoints are point3D_ids[offsets[i] ..
 * offsets[i+1]-1] (DEVICE int64; offsets DEVICE int64 [n_images+1], offsets_host the same values on the HOST, checked
 * non-decreasing); A_i is the set of keypoint INDICES k whose point3D_id is > 0 (an id of 0 counts as missing, as -1).
 * A pack kernel writes bits_out DEVICE uint32 [n_images][words] (bit k % 32 of word k / 32 set iff k is in A_i;
 * words >= ceil(n2d / 32) of every image) and counts_out DEVICE int32 [n_images] = |A_i|.  A count kernel over 64 x 64
 * image tiles of the upper triangle accumulates |A_i ∩ A_j| as int32 popcounts (exact) and writes EVERY entry of
 * scores_out DEVICE double [n_images][n_images]: |A_i ∩ A_j| / max(|A_i|, |A_j|) (one IEEE division) for i < j, 1 on
 * the diagonal, 0 below it.  Two images with empty sets give NaN where the reference raises ZeroDivisionError; the
 * caller checks the counts.  Limits: n_images <= 2^20, n2d < 2^31 per image (words <= 2^26); anything beyond returns
 * -1.  Integer counts: identical across runs. */
P2P_API int p2p_overlap_scores(p2p_handle_t h, const int64_t* point3D_ids, const int64_t* offsets,
                               const int64_t* offsets_host, int n_images, int words, uint32_t* bits_out,
                               int32_t* counts_out, double* scores_out, void* stream);
/* Test hook: hypotheses 0 .. count-1 of p2p_find_model without selection.  models_out DEVICE double [count*slots][9]
 * (slots 3 for F, 1 for H; zero where a slot has no model), counts_out DEVICE int32 [count*slots] (-1: no model). */
P2P_API int p2p_test_hypotheses(p2p_handle_t h, int model, const double* rows, int row_stride, int n, double px_th,
                        unsigned long long seed, int count, double* models_out, int32_t* counts_out, void* stream);
/* Test hook: model 2's degeneracy test on every root of F hypotheses 0 .. count-1 (count <= 2^20), slot layout as
 * p2p_test_hypotheses.  triplet_out DEVICE int32 [count*3]: -2 = no model in the slot, -1 = not degenerate, else the
 * index (0..4) of the first degenerate triplet; H_out DEVICE double [count*3][9]: that triplet's induced H in pixel
 * coordinates at H[2][2] = 1 (zeros unless degenerate). */
P2P_API int p2p_test_degeneracy(p2p_handle_t h, const double* rows, int row_stride, int n, double px_th,
                                unsigned long long seed, int count, int32_t* triplet_out, double* H_out, void* stream);

/* Relative pose -- the reference's matches2relapose_cv (utils/eval/geometry.py:32-48): cv2.findEssentialMat(RANSAC) and
 * cv2.recoverPose, on the device.  rows / row_stride / n / n_dev as p2p_find_model; intr HOST double[8] = (fx1, fy1,
 * cx1, cy1, fx2, fy2, cx2, cy2), focal lengths positive.  Points map to camera coordinates ((x - cx) / fx, (y - cy) / fy).
 *
 * p2p_find_essential: RANSAC for E (x2^T E x1 = 0 in camera coordinates) with the 5-point minimal solver (null space of
 * the 5 x 9 epipolar system, 10 cubic constraints, Gauss-Jordan, Nister's degree-10 polynomial, Sturm bisection; up to
 * 10 models per sample).  Inlier iff the Sampson error in camera coordinates is below th^2, th = px_th / ((fx2 + fy2)
 * / 2) (OpenCV's rule).  Same generator, rounds, stopping bound (s = 5), tie rule and reproducibility as
 * p2p_find_model; the winner is refitted (8-point, projected onto singular values (1, 1, 0)) while the count grows.
 * E_out DEVICE double [9] row-major at unit Frobenius norm, mask_out DEVICE uint8 [n], n_inliers_out DEVICE int32:
 * 0 = no model (E and mask zeroed), -1 = a coordinate is not finite (E NaN, mask zeroed). */
P2P_API int p2p_find_essential(p2p_handle_t h, const double* rows, int row_stride, int n, const double* n_dev,
                               const double* intr, double px_th, double conf, int max_iters, unsigned long long seed,
                               double* E_out, uint8_t* mask_out, int32_t* n_inliers_out, void* stream);
/* p2p_recover_pose: decomposes E (DEVICE double [9]) as cv2.decomposeEssentialMat into [R1|t], [R2|t], [R1|-t],
 * [R2|-t], triangulates every row under mask_in (DEVICE uint8 [n], nullable = all rows) against [I|0] and each
 * candidate, and keeps the candidate with the most points with Q2 Q3 > 0, depth in camera 1 below dist_th and depth in
 * camera 2 in (0, dist_th) (ties to the first).  Rt_out DEVICE double [12]: R row-major then t (unit norm,
 * x2 = R x1 + t); mask_out DEVICE uint8 [n]: the good points; n_good_out DEVICE int32.  A zero or non-finite E gives
 * zero R, t, count and mask. */
P2P_API int p2p_recover_pose(p2p_handle_t h, const double* rows, int row_stride, int n, const double* n_dev,
                             const double* intr, const double* E, const uint8_t* mask_in, double dist_th,
                             double* Rt_out, uint8_t* mask_out, int32_t* n_good_out, void* stream);
/* Test hook: hypotheses 0 .. count-1 of p2p_find_essential without selection.  models_out DEVICE double [count*10][9]
 * (camera coordinates, zero where a slot has no model), counts_out DEVICE int32 [count*10] (-1: no model). */
P2P_API int p2p_test_essential_hypotheses(p2p_handle_t h, const double* rows, int row_stride, int n, const double* intr,
                                          double px_th, unsigned long long seed, int count, double* models_out,
                                          int32_t* counts_out, void* stream);

/* ---- many pairs per call: p2p_find_model / p2p_find_essential / p2p_recover_pose over K pairs, each pair's result
 * bit-identical to the single-pair call on its rows (the same kernels with the pair as one more grid dimension).
 * rows: ONE fp64 row array with one row_stride; pair k owns rows offsets[k] .. offsets[k+1]-1 (offsets DEVICE int64
 * [K+1]; offsets_host the same K+1 values on the HOST).  offsets_host is checked: non-decreasing, from 0 or more, at
 * most 2^26 rows per pair and fewer than 2^31 rows in all (-1 otherwise).  That offsets holds the same values is the
 * caller's contract, as the device-side counts are: it is not read back.  n_dev: DEVICE double [K] or NULL, pair k uses
 * min(n_k, n_dev[k]) rows.  Masks are row-aligned: mask_out (and mask_in) DEVICE uint8 [offsets[K]], pair k's entries
 * at offsets[k] ..; entries of rows before offsets[0] are not touched.  One px_th / conf / max_iters / seed / dist_th
 * serves every pair, so pair k draws exactly the hypotheses of a single-pair call with that seed.  intr: DEVICE double
 * [K][8] as p2p_find_essential's HOST intr; finite values with positive focal lengths are the caller's contract (not
 * read back).  K = 0 enqueues nothing.  Pairs run in launches of at most p2p_batch_chunk_pairs pairs (about 256 MiB of
 * per-pair scratch, and the grid's 65535 limit), one after another on `stream`; the split changes no result.  No host
 * sync. */
P2P_API int p2p_find_model_batch(p2p_handle_t h, int model, const double* rows, int row_stride, const int64_t* offsets,
                                 const int64_t* offsets_host, int K, const double* n_dev, double px_th, double conf,
                                 int max_iters, unsigned long long seed, double* models_out, uint8_t* mask_out,
                                 int32_t* n_inliers_out, void* stream);
/* models_out DEVICE double [K][9], n_inliers_out DEVICE int32 [K]: per pair as p2p_find_model. */
P2P_API int p2p_find_essential_batch(p2p_handle_t h, const double* rows, int row_stride, const int64_t* offsets,
                                     const int64_t* offsets_host, int K, const double* n_dev, const double* intr,
                                     double px_th, double conf, int max_iters, unsigned long long seed, double* E_out,
                                     uint8_t* mask_out, int32_t* n_inliers_out, void* stream);
/* E_out DEVICE double [K][9], n_inliers_out DEVICE int32 [K]: per pair as p2p_find_essential. */
P2P_API int p2p_recover_pose_batch(p2p_handle_t h, const double* rows, int row_stride, const int64_t* offsets,
                                   const int64_t* offsets_host, int K, const double* n_dev, const double* intr,
                                   const double* E, const uint8_t* mask_in, double dist_th, double* Rt_out,
                                   uint8_t* mask_out, int32_t* n_good_out, void* stream);
/* E DEVICE double [K][9], mask_in row-aligned or NULL (all rows), Rt_out DEVICE double [K][12], n_good_out DEVICE int32
 * [K]: per pair as p2p_recover_pose. */
/* p2p_find_essential_batch with one threshold per pair: px_th DEVICE double [K], pair k's px_th (positive and finite
 * are the caller's contract: not read back).  Pair k's result is bit-identical to p2p_find_essential on its rows with
 * px_th[k]; with every entry equal to x it is p2p_find_essential_batch's with px_th = x. */
P2P_API int p2p_find_essential_batch_th(p2p_handle_t h, const double* rows, int row_stride, const int64_t* offsets,
                                        const int64_t* offsets_host, int K, const double* n_dev, const double* intr,
                                        const double* px_th, double conf, int max_iters, unsigned long long seed,
                                        double* E_out, uint8_t* mask_out, int32_t* n_inliers_out, void* stream);
/* The per-pair statistics of the relative-pose evaluation (patch2pix_b200/relpose.py) for K pairs in one launch, no host
 * sync.  rows / row_stride / offsets / offsets_host / n_dev / intr as p2p_find_essential_batch (m_k = min(n_k,
 * n_dev[k]) rows (x1, y1, x2, y2) in columns 0..3).  Rt_gt and Rt_est DEVICE double [K][12]: R row-major then t
 * (x1 = R x0 + t, view 0 -> view 1; t need not be normalised), Rt_est as p2p_recover_pose_batch writes it; n_inliers
 * DEVICE int32 [K], the E-RANSAC inlier counts (<= 0: no model).  thresholds HOST double [n_thr] (1 <= n_thr <= 16,
 * finite, > 0, strictly increasing; anything else returns -1), passed by value to the kernel.  Pair k writes
 * out[k * out_stride ..] (DEVICE, out_stride >= 2 + (n_thr + 2) / 2 doubles):
 *   double [0] = clip((tr(R_gt^T R) - 1) / 2, -1, 1), double [1] = clip(t_gt . t / (|t_gt| |t|), -1, 1), both NaN
 *   when n_inliers[k] <= 0 (the caller takes the arccos, which the device does not round correctly);
 *   then int32 [n_thr + 1] from double 2 on: the rows whose symmetric epipolar error in camera coordinates,
 *   e = (x1^T E x0)^2 (1 / ((E x0)_0^2 + (E x0)_1^2) + 1 / ((E^T x1)_0^2 + (E^T x1)_1^2)) with E = [t_gt]x R_gt and
 *   x = ((x - cx) / fx, (y - cy) / fy, 1), is < thresholds[j] (NaN never is), then m_k.
 * Every fp64 product, sum, quotient and square root is rounded on its own (no fused multiply-add; order in
 * csrc/relpose.cu), so a numpy restatement gives the same bits.  Integer counts: identical across runs and devices. */
P2P_API int p2p_relpose_errors_batch(p2p_handle_t h, const double* rows, int row_stride, const int64_t* offsets,
                                     const int64_t* offsets_host, int K, const double* n_dev, const double* intr,
                                     const double* Rt_gt, const double* Rt_est, const int32_t* n_inliers,
                                     const double* thresholds, int n_thr, double* out, int out_stride, void* stream);
/* Pairs per launch of the batched entry points: entry 0 = p2p_find_model_batch, 1 = p2p_find_essential_batch,
 * 2 = p2p_recover_pose_batch, 3 = p2p_find_absolute_pose_batch (queries). */
P2P_API int p2p_batch_chunk_pairs(p2p_handle_t h, int entry, int* pairs_out);

/* ---- absolute pose from 2D-3D matches (patch2pix_b200/localize.py): RANSAC over K queries in one launch chain, no
 * host sync.  rows: ONE fp64 row array, row = (u, v, X, Y, Z) in columns 0..4 (the pixel in the query, the world
 * point), row_stride >= 5; offsets / offsets_host / n_dev as p2p_find_model_batch (query k owns rows offsets[k] ..
 * offsets[k+1]-1 and uses min(n_k, n_dev[k]) of them).  intr DEVICE double [K][4] = (fx, fy, cx, cy), a pinhole camera
 * without distortion per query (finite, positive focal lengths: the caller's contract, not read back).  px_th_dev
 * DEVICE double [K] (query k's pixel threshold, positive and finite by contract) or NULL: px_th for every query.
 *
 * Per query: the world points are centred on their mean (fp32 scoring stays accurate far from the origin); rounds of
 * 1024 hypotheses draw 3 distinct rows (the p2p_find_model generator) and solve Grunert's P3P quartic in fp64 (Ferrari,
 * two Newton steps per root, up to 4 poses); a row is an inlier iff its depth is > 0 and its squared reprojection
 * error is < px_th^2, scored in fp32.  Selection, tie rule and stopping bound (s = 3) as p2p_find_model.  The winner is
 * refined by Gauss-Newton on the 6-DoF pose over its inliers (3 steps per refit, rotation through the exponential
 * map), each refit kept while the inlier count strictly grows, at most 4 refits.
 * Rt_out DEVICE double [K][12]: R row-major then t, x_cam = R X + t, in world coordinates; mask_out DEVICE uint8,
 * row-aligned; n_inliers_out DEVICE int32 [K].  A query with fewer than 4 rows, or without a model, gets count 0; one
 * with a non-finite value gets -1; both get a NaN pose and a zero mask, and neither affects the other queries.  Query
 * k's result is bit-identical to the same call on its rows alone, and with px_th_dev all equal to x, to the call with
 * px_th = x. */
P2P_API int p2p_find_absolute_pose_batch(p2p_handle_t h, const double* rows, int row_stride, const int64_t* offsets,
                                         const int64_t* offsets_host, int K, const double* n_dev, const double* intr,
                                         double px_th, const double* px_th_dev, double conf, int max_iters,
                                         unsigned long long seed, double* Rt_out, uint8_t* mask_out,
                                         int32_t* n_inliers_out, void* stream);
/* Test hook: hypotheses 0 .. count-1 (count <= 2^20) of one query (n >= 4 rows, intr HOST double [4]) without
 * selection.  models_out DEVICE double [count*4][12]: poses in the centred frame (x_cam = R (X - mean) + t, mean the
 * row-order fixed-tree sum of the world points over n), zero where a slot has none; counts_out DEVICE int32 [count*4]
 * (-1: no pose).  A sample's poses fill its first slots in ascending order of the quartic's root. */
P2P_API int p2p_test_absolute_pose_hypotheses(p2p_handle_t h, const double* rows, int row_stride, int n,
                                              const double* intr, double px_th, unsigned long long seed, int count,
                                              double* models_out, int32_t* counts_out, void* stream);
/* Lift one database cutout's matches to world points (hloc's interpolate_scan + the scan alignment).  scan DEVICE fp64
 * [height][width][3] (the cutout's XYZcut, NaN holes), align HOST double [16] (4x4 row-major, finite), matches DEVICE
 * fp64 rows (xq, yq, xdb, ydb) in columns 0..3, match_stride >= 4, n rows or min(n, *n_dev) (n_dev DEVICE double,
 * nullable).  Per match in order: a database pixel outside [0, width-1] x [0, height-1] (or NaN) is dropped; else the
 * scan is sampled there as grid_sample(align_corners=True) does, bilinear (in-bounds corners only), and a NaN channel
 * takes the nearest pixel's value (round half to even); a point still not finite is dropped; a kept point becomes
 * A[:3, :3] p + A[:3, 3], every product and sum rounded on its own.  Kept rows (xq, yq, X, Y, Z) are written to rows_out
 * (DEVICE, row_stride >= 5) from row *count_dev on, in match order, at most up to row capacity, and *count_dev (DEVICE
 * double: the running count, p2p_find_absolute_pose_batch's n_dev entry) grows by their number.  One block; n = 0
 * enqueues nothing. */
P2P_API int p2p_lift_scan(p2p_handle_t h, const double* scan, int height, int width, const double* align,
                          const double* matches, int match_stride, int n, const double* n_dev, double* rows_out,
                          int row_stride, long long capacity, double* count_dev, void* stream);

/* ---- triangulation against known poses (sfm.cu; the protocol in patch2pix_b200/sfm.py).  All DEVICE arrays unless
 * named HOST; ids come from sorted keys, so every output is independent of grid shape and scheduling.
 *
 * p2p_sfm_keypoints: matches fp64 [n_matches][4] (x0, y0, x1, y1), pair p owning rows offsets[p] .. offsets[p+1]
 * (int64 [n_pairs + 1], offsets[0] = 0), pair_img int32 [n_pairs][2] (image index < 2^20 of each side).  Endpoint e is
 * side e & 1 of match e >> 1 when both_sides, else side 0 of match e.  An endpoint that is not finite, is negative, or
 * whose cell (floor(x / merge_px), floor(y / merge_px)) reaches 2^22 is dropped.  Keypoints are the distinct keys
 * image << 44 | cell_y << 22 | cell_x, ids in key order; kp_xy [.][2] is the mean of the key's endpoints summed in
 * endpoint order, kp_key [.] the key; kp_of_ep [endpoints] the keypoint of each endpoint or -1.  Capacity of the
 * keypoint arrays: the endpoint count.  counts int64 [2] = keypoints, dropped endpoints.  No host sync. */
P2P_API int p2p_sfm_keypoints(p2p_handle_t h, const double* matches, long long n_matches, const int64_t* offsets,
                              int n_pairs, const int32_t* pair_img, int both_sides, double merge_px, double* kp_xy,
                              uint64_t* kp_key, int32_t* kp_of_ep, int64_t* counts, void* stream);
/* Pixels -> undistorted normalised coordinates of keypoints 0 .. min(capacity, *n_dev) - 1 (n_dev nullable): image =
 * kp_key >> 44, camera cams [img_cam[image]] = (model, fx, fy, cx, cy, k1, k2, 0), COLMAP's radial distortion
 * u (1 + k1 r^2 + k2 r^4) inverted by 12 Newton steps from the distorted point. */
P2P_API int p2p_sfm_undistort(p2p_handle_t h, const double* xy, const uint64_t* kp_key, long long capacity,
                              const int64_t* n_dev, const int32_t* img_cam, const double* cams, double* xy_out,
                              void* stream);
/* Edges and tracks of a p2p_sfm_keypoints(both_sides = 1) result.  A match is an edge candidate iff it is the first
 * match of its pair, in match order, for its keypoint on side 0 and also for its keypoint on side 1; it is kept iff
 * its Sampson error under E [n_pairs][9] (row-major, x1^T E x0 = 0 in the normalised coordinates kp_n) is at most
 * thr [n_pairs].  Equal edges collapse.  labels int32 [n_kp]: the smallest keypoint id of each connected component.
 * obs_kp int32 [n_kp]: keypoints sorted by (label, id); a track is a run of 2 .. 2^16 equal labels, track t at
 * obs_kp[track_start[t]] .. + track_len[t] (capacity n_kp), in label order.  counts (DEVICE and HOST int64 [6]) =
 * unique kept edges, tracks, observations in tracks, rejected components over 2^16, first-in-pair matches, 0.
 * Synchronises once (hooking converged), then copies the counts to counts_host. */
P2P_API int p2p_sfm_tracks(p2p_handle_t h, const int32_t* kp_of_ep, long long n_matches, const int64_t* offsets,
                           int n_pairs, const double* E, const double* thr, const double* kp_n, long long n_kp,
                           int32_t* labels, int32_t* obs_kp, int32_t* track_start, int32_t* track_len,
                           int64_t* counts_dev, int64_t* counts_host, void* stream);
/* Multi-view triangulation of each track (rounds of hypotheses, selection, Gauss-Newton, acceptance; sfm.py states
 * them).  images fp64 [.][15] = R row-major, t, centre; cameras as p2p_sfm_undistort; a reprojection error is measured
 * in original (distorted) pixels.  Points are numbered by (track, round): points [.][3], point_len int32 (inlier
 * observations), point_err (their mean error in pixels), capacity n_tracks * 8; kp_point int32 [n_kp] the point of each
 * keypoint or -1.  counts int64 [1] = points.  No host sync. */
P2P_API int p2p_sfm_triangulate(p2p_handle_t h, const int32_t* obs_kp, const int32_t* track_start,
                                const int32_t* track_len, int n_tracks, long long n_kp, const double* kp_xy,
                                const double* kp_n, const uint64_t* kp_key, const double* images,
                                const int32_t* img_cam, const double* cams, double reproj_px, double cos_min_angle,
                                double* points, int32_t* point_len, double* point_err, int32_t* kp_point,
                                int64_t* counts, void* stream);
/* 2D-3D rows of a chunk of queries.  matches / offsets / pair_img as p2p_sfm_keypoints with pair_img = (query index,
 * database image); qkp_* the p2p_sfm_keypoints(both_sides = 0) and p2p_sfm_undistort results of the same matches.
 * Each database endpoint takes the nearest keypoint of its image, among the 3x3 cells around its own, that has a
 * point and lies within merge_px (ties to the lower id); rows fp64 [.][5] = (fx xn + cx, fy yn + cy, X, Y, Z) with
 * q_intr [n_queries][4] = (fx, fy, cx, cy), one per distinct (query keypoint, point), ordered by that pair; q_offsets
 * int64 [n_queries + 1] the rows of each query (the p2p_find_absolute_pose_batch layout).  No host sync. */
P2P_API int p2p_sfm_query_rows(p2p_handle_t h, const double* matches, long long n_matches, const int64_t* offsets,
                               int n_pairs, const int32_t* pair_img, int n_queries, double merge_px,
                               const int32_t* qkp_of_ep, const uint64_t* qkp_key, const double* qkp_n,
                               const double* q_intr, const uint64_t* kp_key, const double* kp_xy,
                               const int32_t* kp_point, long long n_kp, const double* points, double* rows,
                               int64_t* q_offsets, void* stream);

/* ---- SuperPoint keypoints and descriptors, exact nearest-neighbour matching (keypoints.cu; the Python side in
 * patch2pix_b200/superpoint.py, the restatement in oracle/superpoint_oracle.py).
 *
 * p2p_sp_keypoints: logits fp32 [batch][65][hc][wc], the detector head's output.  Per image: softmax over the 65
 * channels, dustbin dropped, depth-to-space to s [H = 8 hc][W = 8 wc] (channel c -> pixel (8 cy + c / 8, 8 cx + c % 8)),
 * written to score_map [batch][H][W] when it is not NULL.  NMS with p = (2 nms_radius + 1)^2 max-pool, stride 1,
 * out-of-image taps never winning: M = (s == p(s)); twice: S = p(M) > 0, s' = S ? 0 : s, M |= (s' == p(s')) & !S.
 * A keypoint is a pixel with (M ? s : 0) > threshold and border <= x < W - border, border <= y < H - border.  With
 * max_keypoints >= 0 an image keeps its min(max_keypoints, count) best by score, descending, exact ties in ascending
 * flat index; with max_keypoints < 0 all, in row-major order.  Output: keypoints fp32 [.][2] (x, y) and scores fp32
 * [.] of all images in image order, and offsets int64 [batch + 1]: image b owns rows offsets[b] .. offsets[b + 1].
 * keypoints / scores hold batch * H * W rows (batch * min(max_keypoints, H * W) with max_keypoints >= 0).
 * Limits: batch * H * W < 2^31, batch <= 65535, hc <= 262140, 0 <= nms_radius <= 16, border >= 0, threshold
 * finite. */
P2P_API int p2p_sp_keypoints(p2p_handle_t h, const float* logits, int batch, int hc, int wc, int nms_radius,
                             float threshold, int border, int max_keypoints, float* score_map, float* keypoints,
                             float* scores, int64_t* offsets, void* stream);
/* p2p_sp_descriptors: desc fp32 [batch][dim][hc][wc], the raw descriptor head; keypoints / offsets as
 * p2p_sp_keypoints wrote them, n = offsets[batch] (HOST value).  Each cell is divided by max(|cell|, 1e-12); a keypoint
 * (x, y) samples that map bilinearly as grid_sample(align_corners=True, zero padding) at
 * gx = (x - 3.5) / (8 wc - 4.5) * 2 - 1 (gy likewise), in fp64; the sample is divided by max(|sample|, 1e-12).
 * Output fp32 [n][dim].  Limits: 1 <= dim <= 512. */
P2P_API int p2p_sp_descriptors(p2p_handle_t h, const float* desc, int batch, int dim, int hc, int wc,
                               const float* keypoints, const int64_t* offsets, long long n, float* out, void* stream);
/* p2p_match_descriptors_batch: n_pairs pairs of descriptor sets, d0 fp32 [.][dim] with pair k's set 0 in rows
 * offsets0[k] .. offsets0[k + 1], d1 and offsets1 likewise (offsets given on the device and, as *_host, on the
 * host).  The similarity of rows i, j is the float64 sum over c = 0 .. dim - 1, in that order, of the exact products
 * d0[i][c] * d1[j][c].  Row i's best column j1 has the largest similarity s1 (ties: lowest j), s2 the largest over the
 * other columns.  Row i is accepted iff the set has a column, and: mutual = 1 -> row i is the best row of column j1
 * (ties: lowest i); min_sim not NaN -> s1 > min_sim; ratio not NaN -> 1 - s1 < ratio * ratio * (1 - s2) in float64,
 * true when the set has one column.  Output per row of d0: match int32 = j1 (pair-local) or -1, sim fp64 = s1 or 0.
 * Results are exact (no tolerance), identical across runs and for a pair alone or in any batch.  Option "match_impl"
 * 1 (default): similarities on the tensor cores (3-pass fp16 hi/lo), every decision within 2 eps of its margin redone
 * in float64 (DESIGN.md); 0: every similarity in float64 on the CUDA cores.  Same result.  Optional outputs (NULL to
 * skip; tensor-core path only): tc_sim [n0] / tc_idx [n0] the tensor-core best similarity and column of each row
 * before the fix-up, eps [n_pairs] the bound of |s_tc - s_fp64| per pair, n_fixed int32 [2] the rows and columns
 * redone in float64.  Limits: 1 <= n_pairs <= 65535, dim % 16 == 0, 16 <= dim <= 1024, fewer than 2^20 rows per set.
 * Descriptors must be finite: a NaN or inf is not detected (that would cost a host sync) and gives unspecified
 * matches. */
P2P_API int p2p_match_descriptors_batch(p2p_handle_t h, const float* d0, const float* d1, const int64_t* offsets0,
                                        const int64_t* offsets1, const int64_t* offsets0_host,
                                        const int64_t* offsets1_host, int n_pairs, int dim, int mutual,
                                        double min_sim, double ratio, int32_t* match, double* sim, double* tc_sim,
                                        int32_t* tc_idx, double* eps, int32_t* n_fixed, void* stream);

/* ---- SuperGlue's optimal transport and match extraction (superglue.cu; the Python side in
 * patch2pix_b200/superglue.py, the float64 restatement in oracle/superglue_oracle.py).
 *
 * p2p_sg_sinkhorn: scores fp32 [batch][n][m], alpha a DEVICE pointer to one fp32 value (SuperGlue's bin_score, read on
 * the device, so the call makes no host sync).  These restate SuperGlue's log_optimal_transport and match extraction:
 *   - couplings C are [n+1][m+1]: scores in the top-left block, alpha in the last row and last column;
 *   - norm = -log(n + m);
 *   - log_mu is norm n times, then log(m) + norm; log_nu is norm m times, then log(n) + norm;
 *   - start with u = v = 0 and run iters times: u_i = log_mu_i - LSE_j(C_ij + v_j), then
 *     v_j = log_nu_j - LSE_i(C_ij + u_i);
 *   - log_assign = C + u_i + v_j - norm, written [batch][n+1][m+1] when log_assign is not NULL.
 * Extraction uses only the top-left n x m block of log_assign:
 *   - i0(i) is the argmax of row i, i1(j) the argmax of column j, ties to the lowest index;
 *   - row i is mutual iff i1(i0(i)) == i (column j likewise);
 *   - mscores0_i = exp(max of row i) if row i is mutual, else 0; mscores1_j = mscores0[i1(j)] if column j is mutual,
 *     else 0;
 *   - valid0_i = mutual_i && mscores0_i > match_threshold; valid1_j = mutual_j && valid0[i1(j)];
 *   - matches0 int32 [batch][n] = valid0 ? i0 : -1, matches1 [batch][m] = valid1 ? i1 : -1;
 *   - mscores0 keeps exp(max) for a mutual row even when it fails the threshold, as SuperGlue does.
 * Any of log_assign, matches0/1, mscores0/1 may be NULL.  fp32 throughout; norm, log_mu and log_nu are rounded to fp32
 * from double.  One warp computes each u_i / v_j in a fixed order, so results are bit-identical for any grid size
 * (option "num_sms") and pair k of a batch equals its single-pair call.  One cooperative launch; scratch is a transposed
 * copy of the scores (4 batch n m bytes) plus O(batch (n + m)), grow-only in the handle: after the first call of a
 * shape the call makes no host sync.  Limits: batch, n, m >= 1, n, m <= 2^20, batch (n + 1) (m + 1) < 2^31,
 * 0 <= iters <= 100000, match_threshold finite.  Scores and alpha must be finite: a NaN or inf is not detected (that
 * would cost a host sync) and gives unspecified results.  A failed cooperative launch returns its error. */
P2P_API int p2p_sg_sinkhorn(p2p_handle_t h, const float* scores, int batch, int n, int m, const float* alpha,
                            int iters, float match_threshold, float* log_assign, int32_t* matches0, int32_t* matches1,
                            float* mscores0, float* mscores1, void* stream);

/* ---- bring-up / accuracy probe: C[M,N] = alpha * A[M,K] B[N,K]^T on the wgmma path with the
 * same operand format as the hot path (fp32 inputs are split to fp16 hi/lo on the device).
 * a, b, c are DEVICE fp32; K % 64 == 0. */
P2P_API int p2p_test_gemm(p2p_handle_t h, const float* a, const float* b, float* c, int M, int N, int K, int passes,
                  int seg_len, float in_scale, void* stream);

/* ---- per-tile phase trace (option "tile_trace"): traced launch idx (0 .. "tile_traces" - 1) in launch order.  tag:
 * stage * 8 + kind, stage 0 mid, 1 fine, 2 risk band; kind 0 conv1, 1 shared-window prefix, 2 continuation,
 * 3 unshared rows, 4 conv2; tag 24 = p2p_test_gemm.  tiles: an upper bound of the launch's tiles.  out (optional,
 * host, max_tiles >= tiles): 8 %globaltimer ns stamps per tile -- 0 producer's first load issued, 1 consumer tile
 * start, 2 first stage ready, 3 last k-step issued, 4 accumulators drained, 5 epilogue done, 6 CTA index + 1 -- all
 * zero for tiles the launch did not have.  Synchronises the device. */
P2P_API int p2p_tile_trace_read(p2p_handle_t h, int idx, int* tag, int* tiles, unsigned long long* out, int max_tiles);

#ifdef __cplusplus
}
#endif
#endif /* P2P_B200_H_ */
