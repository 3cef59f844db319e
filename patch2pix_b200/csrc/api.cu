// C ABI of libp2p_b200.so (declared in include/p2p_b200.h): handle, weight packing, stage drivers.
#include <math.h>
#include <stdlib.h>

#include <algorithm>
#include <vector>

#include "../../include/p2p_b200.h"
#include "kernels.h"
#include "umma_gemm.h"

namespace p2p {

static thread_local std::string g_last_error;
void set_last_error(const std::string& msg) { g_last_error = msg; }
long long g_launch_count = 0;

int ensure_dyn_smem(const void* kernel, int bytes) {
  struct Key { const void* k; int dev; };
  static thread_local std::vector<std::pair<Key, int>> granted;
  int dev = 0;
  cudaGetDevice(&dev);
  for (auto& g : granted)
    if (g.first.k == kernel && g.first.dev == dev) {
      if (g.second >= bytes) return 0;
      if (cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes) != cudaSuccess) {
        set_last_error(std::string("cudaFuncSetAttribute(MaxDynamicSharedMemorySize) failed: ") + cudaGetErrorString(cudaGetLastError()));
        return -2;
      }
      g.second = bytes;
      return 0;
    }
  if (cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes) != cudaSuccess) {
    set_last_error(std::string("cudaFuncSetAttribute(MaxDynamicSharedMemorySize) failed: ") + cudaGetErrorString(cudaGetLastError()));
    return -2;
  }
  granted.push_back({Key{kernel, dev}, bytes});
  return 0;
}

int Arena::reserve(size_t bytes) {
  off = 0;
  if (bytes <= cap) return 0;
  if (base != nullptr) {
    cudaDeviceSynchronize();
    cudaFree(base);
    base = nullptr;
    cap = 0;
  }
  bytes = align_up(bytes + (bytes >> 3), 1 << 20);
  if (cudaMalloc(&base, bytes) != cudaSuccess) {
    cudaGetLastError();
    set_last_error("out of device memory reserving " + std::to_string(bytes >> 20) + " MiB of scratch");
    return -3;
  }
  cap = bytes;
  return 0;
}
void Arena::release() {
  if (base != nullptr) cudaFree(base);
  base = nullptr;
  cap = off = 0;
}

struct Regressor {
  bool set = false;
  __half *w1_hi = nullptr, *w1_lo = nullptr;  // [512][73*64]
  __half *w2_hi = nullptr, *w2_lo = nullptr;  // [512][72*64]
  float *scale1 = nullptr, *bias1 = nullptr, *scale2 = nullptr, *bias2 = nullptr;
  float y_scale = 1.f;
  FcWeights fc = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
  // tensor-core FC path: K-major fp16 hi/lo weights [out][in] with per-row pow2 scale, 1/(act*w scale), bias
  __half *f1_hi = nullptr, *f1_lo = nullptr, *f2_hi = nullptr, *f2_lo = nullptr;
  float *fa1 = nullptr, *fa2 = nullptr;
  float fc_scale[3] = {1.f, 1.f, 1.f};   // power-of-two scales of the FC operands: pooled, h1, h2
  KStep steps1[kConv1Steps];
  KStep steps2[kConv2Steps];
  KStep *d_steps1 = nullptr, *d_steps2 = nullptr;
  char* blob = nullptr;  // one allocation backing all of the above
};

}  // namespace p2p

using namespace p2p;

struct p2p_handle_s {
  int device = 0;
  int num_sms = 132;
  int opt_mid_passes = 3, opt_fine_passes = 1, opt_corr_passes = 3, opt_seg_len = 3, opt_gemm_impl = 0, opt_num_sms = 0;
  int opt_mid_band = 26;  // thousandths of a pixel (2x the largest 1-pass/3-pass mid difference over 125k distinct coordinates);
                          // 0 = pure 3-pass mid stage
  int opt_fc_impl = 1;      // 1: the two big Linear layers on the tensor cores (3-pass); 0: CUDA-core FC kernel
  int opt_fuse_gather = 3;  // conv1 A operand of the 1-pass launches: 3 (default): strided TMA boxes of a per-image window map
                            // (AMODE_WINDOW); 1 or 2: gathered by producer warps (AMODE_GATHER); 0: separate gather kernel +
                            // TMA of the patch tensor
  int opt_share_windows = 1;  // mid stage, fuse_gather = 3, 1-pass: compute the conv1 half of an anchor window that a
                              // half-group of 4 rows shares once (1, default), or every row's whole conv1 (0)
  int opt_epi_async = 1;      // 256-wide conv1 / conv2 launches: epilogue straight from the wgmma fragments, conv1's
                              // fp16 tile out by TMA store (1, default), or through the fp32 staging buffer (0); same bits
  int frag_epi_launches = 0;  // conv launches run with the fragment epilogues so far
  int opt_tile_trace = 0;     // 1: every umma_gemm launch of run_regressor / p2p_test_gemm records its per-tile phase trace
  unsigned long long* trace_buf = nullptr;   // device, kTraceCap stamps
  size_t trace_used = 0;
  struct TraceRec {
    int tag, tiles;
    size_t off;
  };
  std::vector<TraceRec> traces;               // the traced launches since tile_trace was last set
  const int* last_band_count = nullptr;  // device counter of the last risk-band subset
  int* share_rows = nullptr;             // device: rows that shared a window half in the last sharing mid-stage call
  bool last_mid_shared = false;          // the last mid-stage call shared windows (share_rows is its count)
  unsigned long long* band_totals = nullptr;   // device: {band rows, rows} summed over mid-stage calls
  struct RefineTap {            // the buffers of the last p2p_refine call's last pass (p2p_refine_taps)
    const __half *y_hi = nullptr, *y_lo = nullptr, *h1_hi = nullptr, *h1_lo = nullptr, *h2_hi = nullptr, *h2_lo = nullptr;
    const float *pooled = nullptr, *raw = nullptr;
    const int *rowmap = nullptr, *d_count = nullptr;   // risk-band subset: slot -> row, and the slot count
    int n = 0, passes = 0, fc_tc = 0;
    float scales[4] = {1.f, 1.f, 1.f, 1.f};            // y_scale, then the pooled, h1 and h2 operand scales
  } tap;
  bool nc_set = false;
  float *nc_w1p = nullptr, *nc_b1p = nullptr, *nc_w2p = nullptr;
  float nc_b2 = 0.f;
  NcUmmaWeights ncw;            // tensor-core NC operand images
  NcStackWeights ncs;           // general NeighConsensus stack (p2p_set_nc_stack_weights), beside the fixed stack above
  bool ncs_set = false;
  void* dbg_nc[4] = {nullptr, nullptr, nullptr, nullptr};   // scratch of the last p2p_neigh_consensus call (debug hook below)
  int opt_match_impl = 1;       // p2p_match_descriptors_batch: 1 tensor-core pass + float64 fix-up, 0 float64 only
  int opt_unique_impl = 1;      // 1: rank sort over the whole GPU for lists <= 8192 rows; 0: single-block bitonic network
  int* uniq_rank = nullptr;     // zeroed scratch of the rank-sort path
  int opt_nc_l2_mode = 0;       // NC layer 2 block layout: 0 auto, 1 one haloed block per tile, 2 one block per column tap
  int opt_nc_impl = 1;          // 1: NeighConsensus on the tensor cores (nc_umma.cu); 0: fp32 CUDA-core kernels (shape-capped)
  Regressor reg[2];
  Arena coarse, refine, feat, misc, uniq, pre, verify, sfm, sp, sg;
  std::vector<PreprocessCoefs> pre_coefs;   // cached resampling tables, one per image geometry
  PairFeatures pf[2];
  bool prepared = false;
  // optional per-kernel CUDA-event profile (p2p_set_option("profile", 1))
  int opt_profile = 0;
  struct ProfEntry { cudaEvent_t a, b; int kind; };
  std::vector<ProfEntry> prof;
  std::vector<cudaEvent_t> event_pool;
};

namespace {

struct DeviceGuard {
  int prev = -1;
  bool ok = true;
  explicit DeviceGuard(int dev) {
    if (cudaGetDevice(&prev) != cudaSuccess) ok = false;
    if (ok && prev != dev && cudaSetDevice(dev) != cudaSuccess) ok = false;
  }
  ~DeviceGuard() {
    if (prev >= 0) cudaSetDevice(prev);
  }
};

#define P2P_ENTER(h)                                                  \
  P2P_REQUIRE((h) != nullptr, "null handle");                         \
  DeviceGuard _guard((h)->device);                                    \
  if (!_guard.ok) {                                                   \
    set_last_error("cannot select CUDA device of the handle");        \
    return -2;                                                        \
  }

float pow2_floor_scale(float maxabs, float target_hi) {
  // power of two s such that maxabs * s lies in [target_hi/2, target_hi)
  if (!(maxabs > 0.f) || !isfinite(maxabs)) return 1.f;
  int e;
  frexpf(maxabs, &e);  // maxabs = m * 2^e, m in [0.5,1)
  int et;
  frexpf(target_hi, &et);
  return ldexpf(1.f, et - 1 - e);
}

void split_half(float v, __half& hi, __half& lo) {
  hi = __float2half_rn(v);
  lo = __float2half_rn(v - __half2float(hi));
}

template <typename T>
T* carve(char*& p, size_t count) {
  T* r = reinterpret_cast<T*>(p);
  p += align_up(count * sizeof(T), 256);
  return r;
}

void fold_bn(const p2p_bn_t& bn, int n, float eps, std::vector<float>& g, std::vector<float>& b) {
  g.resize(n);
  b.resize(n);
  for (int i = 0; i < n; ++i) {
    g[i] = bn.weight[i] / sqrtf(bn.running_var[i] + eps);
    b[i] = bn.bias[i] - bn.running_mean[i] * g[i];
  }
}

int tap_plane(int t, int& start) {  // conv1 tap -> (parity plane bit, box start)
  if (t == 0) { start = -1; return 0; }
  if (t == 1) { start = 0; return 1; }
  start = 0;
  return 0;
}

int pack_regressor(p2p_handle_s* h, Regressor& R, const p2p_regressor_weights_t& w) {
  const int K1 = kConv1Steps * 64, K2 = kConv2Steps * 64;
  std::vector<float> g1, b1, g2, b2, gf1, bf1, gf2, bf2;
  fold_bn(w.conv1_bn, 512, w.bn_eps, g1, b1);
  fold_bn(w.conv3_bn, 512, w.bn_eps, g2, b2);
  fold_bn(w.fc1_bn, 512, w.bn_eps, gf1, bf1);
  fold_bn(w.fc4_bn, 256, w.bn_eps, gf2, bf2);

  std::vector<__half> w1h((size_t)512 * K1), w1l((size_t)512 * K1), w2h((size_t)512 * K2), w2l((size_t)512 * K2);
  std::vector<float> sc1(512), sc2(512), bi1(b1), bi2(b2);
  float max_bound = 0.f;
  std::vector<float> sw1(512), sw2(512);
  std::vector<double> ybound(512);   // |conv1 output| of each channel, for any L2-normalised input
  for (int o = 0; o < 512; ++o) {
    const float* wo = w.conv0_weight + (size_t)o * 518 * 9;
    float m = 0.f;
    double tapn[9] = {0};
    for (int c = 0; c < 518; ++c)
      for (int t = 0; t < 9; ++t) {
        const float v = wo[c * 9 + t] * g1[o];
        m = fmaxf(m, fabsf(v));
        tapn[t] += (double)v * v;
      }
    float bound = fabsf(b1[o]);
    for (int t = 0; t < 9; ++t) bound += 1.41421357f * (float)sqrt(tapn[t]);
    max_bound = fmaxf(max_bound, bound);
    ybound[o] = bound;
    sw1[o] = pow2_floor_scale(m, 1024.f);
    sc1[o] = 1.f / (kActScale * sw1[o]);
    __half* dh = w1h.data() + (size_t)o * K1;
    __half* dl = w1l.data() + (size_t)o * K1;
    for (int s = 0; s < 72; ++s) {
      const int tap = s / 8, chunk = s % 8;
      for (int kk = 0; kk < 64; ++kk) {
        const int c512 = chunk * 64 + kk;
        const int orig = (c512 / 256) * 259 + 3 + (c512 % 256);
        split_half(wo[orig * 9 + tap] * g1[o] * sw1[o], dh[s * 64 + kk], dl[s * 64 + kk]);
      }
    }
    for (int kk = 0; kk < 64; ++kk) {
      float v = 0.f;
      if (kk < 54) {
        const int tap = kk / 6, r = kk % 6;
        const int orig = (r / 3) * 259 + (r % 3);
        v = wo[orig * 9 + tap] * g1[o] * sw1[o];
      }
      split_half(v, dh[72 * 64 + kk], dl[72 * 64 + kk]);
    }
  }
  R.y_scale = pow2_floor_scale(max_bound, 32768.f);
  for (int o = 0; o < 512; ++o) {
    const float* wo = w.conv2_weight + (size_t)o * 512 * 9;
    float m = 0.f;
    for (int i = 0; i < 512 * 9; ++i) m = fmaxf(m, fabsf(wo[i] * g2[o]));
    sw2[o] = pow2_floor_scale(m, 1024.f);
    sc2[o] = 1.f / (R.y_scale * sw2[o]);
    __half* dh = w2h.data() + (size_t)o * K2;
    __half* dl = w2l.data() + (size_t)o * K2;
    for (int s = 0; s < 72; ++s) {
      const int tap = s / 8, chunk = s % 8;
      for (int kk = 0; kk < 64; ++kk)
        split_half(wo[(chunk * 64 + kk) * 9 + tap] * g2[o] * sw2[o], dh[s * 64 + kk], dl[s * 64 + kk]);
    }
  }
  // k-step plans
  for (int s = 0; s < 72; ++s) {
    const int tap = s / 8, chunk = s % 8, ty = tap / 3, tx = tap % 3;
    int sx, sy;
    const int px = tap_plane(tx, sx), py = tap_plane(ty, sy);
    R.steps1[s] = KStep{(short)(chunk * 64), (signed char)sx, (signed char)sy, (signed char)(py * 2 + px), 0, 0, s * 64};
    R.steps2[s] = KStep{(short)(chunk * 64), (signed char)(tx - 1), (signed char)(ty - 1), 0, 0, 0, s * 64};
  }
  R.steps1[72] = KStep{0, 0, 0, 0, 1, 0, 72 * 64};
  // FC (BN folded, transposed)
  std::vector<float> f1t((size_t)512 * 512), f1b(512), f2t((size_t)512 * 256), f2b(256), f3t(256 * 5), f3b(5);
  for (int o = 0; o < 512; ++o) {
    for (int k = 0; k < 512; ++k) f1t[(size_t)k * 512 + o] = w.fc0_weight[(size_t)o * 512 + k] * gf1[o];
    f1b[o] = w.fc0_bias[o] * gf1[o] + bf1[o];
  }
  for (int o = 0; o < 256; ++o) {
    for (int k = 0; k < 512; ++k) f2t[(size_t)k * 256 + o] = w.fc3_weight[(size_t)o * 512 + k] * gf2[o];
    f2b[o] = w.fc3_bias[o] * gf2[o] + bf2[o];
  }
  for (int o = 0; o < 5; ++o) {
    for (int k = 0; k < 256; ++k) f3t[k * 5 + o] = w.fc6_weight[o * 256 + k];
    f3b[o] = w.fc6_bias[o];
  }
  // Activation bounds of the FC operands, continuing conv1's: pooled[o] = max relu(conv2) <= P[o] (conv1 outputs of
  // either sign), h1[o] = relu(bias + W1 pooled) <= relu(bias + sum_k max(W1[o][k], 0) P[k]) as pooled >= 0, h2 likewise
  // from h1 >= 0.  Each operand is scaled by the power of two that puts its bound in [2^14, 2^15), so the fp16 hi
  // part never saturates (the epilogues' clip at 65504 stays out of reach) while O(1) activations keep their lo bits.
  std::vector<double> pb(512), h1b(512), h2b(256);
  for (int o = 0; o < 512; ++o) {
    const float* wo = w.conv2_weight + (size_t)o * 512 * 9;
    double a = b2[o];
    for (int c = 0; c < 512; ++c)
      for (int t = 0; t < 9; ++t) a += fabs((double)wo[c * 9 + t] * g2[o]) * ybound[c];
    pb[o] = std::max(a, 0.0);
  }
  for (int o = 0; o < 512; ++o) {
    double a = f1b[o];
    for (int k = 0; k < 512; ++k) a += std::max((double)f1t[(size_t)k * 512 + o], 0.0) * pb[k];
    h1b[o] = std::max(a, 0.0);
  }
  for (int o = 0; o < 256; ++o) {
    double a = f2b[o];
    for (int k = 0; k < 512; ++k) a += std::max((double)f2t[(size_t)k * 256 + o], 0.0) * h1b[k];
    h2b[o] = std::max(a, 0.0);
  }
  const float fc_bound[3] = {(float)*std::max_element(pb.begin(), pb.end()), (float)*std::max_element(h1b.begin(), h1b.end()),
                             (float)*std::max_element(h2b.begin(), h2b.end())};
  for (int i = 0; i < 3; ++i) R.fc_scale[i] = pow2_floor_scale(fc_bound[i], 32768.f);
  // tensor-core FC operands
  std::vector<__half> f1h((size_t)512 * 512), f1l((size_t)512 * 512), f2h((size_t)256 * 512), f2l((size_t)256 * 512);
  std::vector<float> fa1(512), fa2(256);
  for (int o = 0; o < 512; ++o) {
    float m = 0.f;
    for (int k = 0; k < 512; ++k) m = fmaxf(m, fabsf(w.fc0_weight[(size_t)o * 512 + k] * gf1[o]));
    const float sw = pow2_floor_scale(m, 1024.f);
    fa1[o] = 1.f / (R.fc_scale[0] * sw);
    for (int k = 0; k < 512; ++k)
      split_half(w.fc0_weight[(size_t)o * 512 + k] * gf1[o] * sw, f1h[(size_t)o * 512 + k], f1l[(size_t)o * 512 + k]);
  }
  for (int o = 0; o < 256; ++o) {
    float m = 0.f;
    for (int k = 0; k < 512; ++k) m = fmaxf(m, fabsf(w.fc3_weight[(size_t)o * 512 + k] * gf2[o]));
    const float sw = pow2_floor_scale(m, 1024.f);
    fa2[o] = 1.f / (R.fc_scale[1] * sw);
    for (int k = 0; k < 512; ++k)
      split_half(w.fc3_weight[(size_t)o * 512 + k] * gf2[o] * sw, f2h[(size_t)o * 512 + k], f2l[(size_t)o * 512 + k]);
  }
  // device blob
  const size_t total = 2 * 1024 * 1024 + 65536 + 4 * align_up((size_t)512 * K1 * 2, 256) + 8 * 4096 + align_up(f1t.size() * 4, 256) +
                       align_up(f2t.size() * 4, 256) + 8 * 8192 + 65536;
  if (R.blob == nullptr) {
    if (cudaMalloc(&R.blob, total) != cudaSuccess) {
      cudaGetLastError();
      set_last_error("out of device memory packing regressor weights");
      return -3;
    }
  }
  char* p = R.blob;
  R.w1_hi = carve<__half>(p, (size_t)512 * K1);
  R.w1_lo = carve<__half>(p, (size_t)512 * K1);
  R.w2_hi = carve<__half>(p, (size_t)512 * K2);
  R.w2_lo = carve<__half>(p, (size_t)512 * K2);
  R.scale1 = carve<float>(p, 512);
  R.bias1 = carve<float>(p, 512);
  R.scale2 = carve<float>(p, 512);
  R.bias2 = carve<float>(p, 512);
  R.fc.w1t = carve<float>(p, f1t.size());
  R.fc.b1 = carve<float>(p, 512);
  R.fc.w2t = carve<float>(p, f2t.size());
  R.fc.b2 = carve<float>(p, 256);
  R.fc.w3t = carve<float>(p, f3t.size());
  R.fc.b3 = carve<float>(p, 5);
  R.d_steps1 = carve<KStep>(p, kConv1Steps);
  R.d_steps2 = carve<KStep>(p, kConv2Steps);
  R.f1_hi = carve<__half>(p, f1h.size());
  R.f1_lo = carve<__half>(p, f1l.size());
  R.f2_hi = carve<__half>(p, f2h.size());
  R.f2_lo = carve<__half>(p, f2l.size());
  R.fa1 = carve<float>(p, 512);
  R.fa2 = carve<float>(p, 256);
#define UP(dst, src, bytes) P2P_CUDA_OK(cudaMemcpy(dst, src, bytes, cudaMemcpyHostToDevice))
  UP(R.w1_hi, w1h.data(), w1h.size() * 2);
  UP(R.w1_lo, w1l.data(), w1l.size() * 2);
  UP(R.w2_hi, w2h.data(), w2h.size() * 2);
  UP(R.w2_lo, w2l.data(), w2l.size() * 2);
  UP(R.scale1, sc1.data(), 2048);
  UP(R.bias1, bi1.data(), 2048);
  UP(R.scale2, sc2.data(), 2048);
  UP(R.bias2, bi2.data(), 2048);
  UP(R.fc.w1t, f1t.data(), f1t.size() * 4);
  UP(R.fc.b1, f1b.data(), 2048);
  UP(R.fc.w2t, f2t.data(), f2t.size() * 4);
  UP(R.fc.b2, f2b.data(), 1024);
  UP(R.fc.w3t, f3t.data(), f3t.size() * 4);
  UP(R.fc.b3, f3b.data(), 20);
  UP(R.d_steps1, R.steps1, sizeof(R.steps1));
  UP(R.d_steps2, R.steps2, sizeof(R.steps2));
  UP(R.f1_hi, f1h.data(), f1h.size() * 2);
  UP(R.f1_lo, f1l.data(), f1l.size() * 2);
  UP(R.f2_hi, f2h.data(), f2h.size() * 2);
  UP(R.f2_lo, f2l.data(), f2l.size() * 2);
  UP(R.fa1, fa1.data(), 2048);
  UP(R.fa2, fa2.data(), 1024);
#undef UP
  R.set = true;
  (void)h;
  return 0;
}

int sms(const p2p_handle_s* h) { return h->opt_num_sms > 0 ? h->opt_num_sms : h->num_sms; }

constexpr size_t kTraceCap = (size_t)8 << 20;   // stamps (64 MB)

// tile_trace: points p.trace at a zeroed region of the trace buffer for this launch (tag: see p2p_tile_trace_read), or
// leaves it null when tracing is off or the buffer is full
int set_trace(p2p_handle_s* h, UmmaGemmParams& p, int tag, cudaStream_t st) {
  p.trace = nullptr;
  if (!h->opt_tile_trace) return 0;
  const int tiles = p.m_tiles * p.n_tiles * 2;   // an upper bound for 128- and 256-wide tiles
  const size_t need = (size_t)tiles * kTraceStamps;
  if (h->trace_buf == nullptr) P2P_CUDA_OK(cudaMalloc(&h->trace_buf, kTraceCap * sizeof(unsigned long long)));
  if (h->trace_used + need > kTraceCap) return 0;
  p.trace = h->trace_buf + h->trace_used;
  P2P_CUDA_OK(cudaMemsetAsync(p.trace, 0, need * sizeof(unsigned long long), st));
  h->traces.push_back({tag, tiles, h->trace_used});
  h->trace_used += need;
  return 0;
}

// Brackets a group of launches with CUDA events on the launching stream when profiling is on.
struct ProfScope {
  p2p_handle_s* h;
  cudaStream_t st;
  cudaEvent_t a = nullptr, b = nullptr;
  int kind;
  static cudaEvent_t get(p2p_handle_s* h) {
    if (!h->event_pool.empty()) {
      cudaEvent_t e = h->event_pool.back();
      h->event_pool.pop_back();
      return e;
    }
    cudaEvent_t e = nullptr;
    cudaEventCreate(&e);
    return e;
  }
  ProfScope(p2p_handle_s* h_, int kind_, cudaStream_t st_) : h(h_), st(st_), kind(kind_) {
    if (h->opt_profile) {
      a = get(h);
      b = get(h);
      cudaEventRecord(a, st);
    }
  }
  ~ProfScope() {
    if (a != nullptr) {
      cudaEventRecord(b, st);
      h->prof.push_back({a, b, kind});
    }
  }
};

}  // namespace

extern "C" {

const char* p2p_last_error(void) { return g_last_error.c_str(); }
int p2p_version(void) { return 100; }

int p2p_create(int device, p2p_handle_t* out) {
  P2P_REQUIRE(out != nullptr, "out is null");
  int ndev = 0;
  P2P_CUDA_OK(cudaGetDeviceCount(&ndev));
  P2P_REQUIRE(device >= 0 && device < ndev, "device index out of range");
  cudaDeviceProp prop;
  P2P_CUDA_OK(cudaGetDeviceProperties(&prop, device));
  if (prop.major != 9 || prop.minor != 0) {
    set_last_error(std::string("libp2p_b200 targets sm_90a (H100) only; device is sm_") + std::to_string(prop.major) +
                   std::to_string(prop.minor));
    return -2;
  }
  p2p_handle_s* h = new p2p_handle_s();
  h->device = device;
  h->num_sms = prop.multiProcessorCount;
  {
    DeviceGuard g(device);
    if (cudaMalloc(&h->band_totals, 2 * sizeof(unsigned long long)) == cudaSuccess)
      cudaMemset(h->band_totals, 0, 2 * sizeof(unsigned long long));
    else
      h->band_totals = nullptr;
    if (cudaMalloc(&h->share_rows, sizeof(int)) == cudaSuccess)
      cudaMemset(h->share_rows, 0, sizeof(int));
    else
      h->share_rows = nullptr;
  }
  *out = h;
  return 0;
}

int p2p_destroy(p2p_handle_t h) {
  if (h == nullptr) return 0;
  DeviceGuard g(h->device);
  cudaDeviceSynchronize();
  h->coarse.release();
  h->refine.release();
  h->feat.release();
  h->misc.release();
  h->uniq.release();
  h->pre.release();
  h->verify.release();
  h->sfm.release();
  h->sp.release();
  h->sg.release();
  for (auto& c : h->pre_coefs)
    if (c.d) cudaFree(c.d);
  for (auto& e : h->prof) { cudaEventDestroy(e.a); cudaEventDestroy(e.b); }
  for (auto e : h->event_pool) cudaEventDestroy(e);
  if (h->nc_w1p) cudaFree(h->nc_w1p);
  if (h->ncw.blob) cudaFree(h->ncw.blob);
  nc_stack_release(h->ncs);
  if (h->band_totals) cudaFree(h->band_totals);
  if (h->share_rows) cudaFree(h->share_rows);
  if (h->trace_buf) cudaFree(h->trace_buf);
  if (h->uniq_rank) cudaFree(h->uniq_rank);
  for (int i = 0; i < 2; ++i)
    if (h->reg[i].blob) cudaFree(h->reg[i].blob);
  delete h;
  return 0;
}

int p2p_set_ncn_weights(p2p_handle_t h, const float* w1, const float* b1, const float* w2, const float* b2) {
  P2P_ENTER(h);
  P2P_REQUIRE(w1 && b1 && w2 && b2, "null weight pointer");
  // reference layout [k1][Cout][Cin][k2][k3][k4]; logical W[o][c][a][b][d][e] = weight[a][o][c][b][d][e]
  std::vector<float> w1p(81 * 32), b1p(32), w2p(81 * 32);
  for (int a = 0; a < 3; ++a)
    for (int b = 0; b < 3; ++b)
      for (int d = 0; d < 3; ++d)
        for (int e = 0; e < 3; ++e) {
          const int tap = ((a * 3 + b) * 3 + d) * 3 + e;
          for (int c = 0; c < 16; ++c) {
            // net 0: plain weights; net 1: (a,b) <-> (d,e) swapped (the "transposed" pass)
            w1p[tap * 32 + c] = w1[((a * 16 + c) * 1 + 0) * 27 + (b * 3 + d) * 3 + e];
            w1p[tap * 32 + 16 + c] = w1[((d * 16 + c) * 1 + 0) * 27 + (e * 3 + a) * 3 + b];
            w2p[tap * 32 + c] = w2[((a * 1 + 0) * 16 + c) * 27 + (b * 3 + d) * 3 + e];
            w2p[tap * 32 + 16 + c] = w2[((d * 1 + 0) * 16 + c) * 27 + (e * 3 + a) * 3 + b];
          }
        }
  for (int c = 0; c < 16; ++c) b1p[c] = b1p[16 + c] = b1[c];
  if (h->nc_w1p == nullptr) P2P_CUDA_OK(cudaMalloc(&h->nc_w1p, sizeof(float) * (81 * 32 * 2 + 32)));
  h->nc_w2p = h->nc_w1p + 81 * 32;
  h->nc_b1p = h->nc_w2p + 81 * 32;
  P2P_CUDA_OK(cudaMemcpy(h->nc_w1p, w1p.data(), sizeof(float) * 81 * 32, cudaMemcpyHostToDevice));
  P2P_CUDA_OK(cudaMemcpy(h->nc_w2p, w2p.data(), sizeof(float) * 81 * 32, cudaMemcpyHostToDevice));
  P2P_CUDA_OK(cudaMemcpy(h->nc_b1p, b1p.data(), sizeof(float) * 32, cudaMemcpyHostToDevice));
  h->nc_b2 = b2[0];
  {
    int rc = nc_umma_pack(w1p.data(), b1p.data(), w2p.data(), h->ncw);
    if (rc) return rc;
  }
  h->nc_set = true;
  return 0;
}

int p2p_set_nc_stack_weights(p2p_handle_t h, int n_layers, const int* kernel_sizes, const int* channels,
                              const float* const* weights, const float* const* biases, int symmetric) {
  P2P_ENTER(h);
  P2P_REQUIRE(kernel_sizes && channels && weights && biases, "null argument");
  int rc = nc_stack_pack(n_layers, kernel_sizes, channels, weights, biases, symmetric, h->ncs);
  if (rc) return rc;
  h->ncs_set = true;
  return 0;
}

int p2p_set_regressor_weights(p2p_handle_t h, int which, const p2p_regressor_weights_t* w) {
  P2P_ENTER(h);
  P2P_REQUIRE(which == 0 || which == 1, "which must be 0 (mid) or 1 (fine)");
  P2P_REQUIRE(w != nullptr && w->conv0_weight && w->conv2_weight && w->fc0_weight && w->fc3_weight && w->fc6_weight,
              "null weight pointer");
  return pack_regressor(h, h->reg[which], *w);
}

static int* option_slot(p2p_handle_t h, const char* key) {
  if (!strcmp(key, "mid_passes")) return &h->opt_mid_passes;
  if (!strcmp(key, "fine_passes")) return &h->opt_fine_passes;
  if (!strcmp(key, "corr_passes")) return &h->opt_corr_passes;
  if (!strcmp(key, "seg_len")) return &h->opt_seg_len;
  if (!strcmp(key, "gemm_impl")) return &h->opt_gemm_impl;
  if (!strcmp(key, "num_sms")) return &h->opt_num_sms;
  if (!strcmp(key, "profile")) return &h->opt_profile;
  if (!strcmp(key, "mid_band")) return &h->opt_mid_band;
  if (!strcmp(key, "fuse_gather")) return &h->opt_fuse_gather;
  if (!strcmp(key, "share_windows")) return &h->opt_share_windows;
  if (!strcmp(key, "epi_async")) return &h->opt_epi_async;
  if (!strcmp(key, "tile_trace")) return &h->opt_tile_trace;
  if (!strcmp(key, "fc_impl")) return &h->opt_fc_impl;
  if (!strcmp(key, "nc_impl")) return &h->opt_nc_impl;
  if (!strcmp(key, "nc_l2_mode")) return &h->opt_nc_l2_mode;
  if (!strcmp(key, "unique_impl")) return &h->opt_unique_impl;
  if (!strcmp(key, "match_impl")) return &h->opt_match_impl;
  return nullptr;
}

int p2p_set_option(p2p_handle_t h, const char* key, int value) {
  P2P_REQUIRE(h != nullptr && key != nullptr, "null argument");
  int* s = option_slot(h, key);
  P2P_REQUIRE(s != nullptr, std::string("unknown option ") + key);
  if (s == &h->opt_mid_passes || s == &h->opt_fine_passes) P2P_REQUIRE(value == 1 || value == 3, "passes must be 1 or 3");
  if (s == &h->opt_corr_passes) P2P_REQUIRE(value == 0 || value == 1 || value == 3, "corr_passes must be 0, 1 or 3");
  if (s == &h->opt_share_windows) P2P_REQUIRE(value == 0 || value == 1, "share_windows must be 0 or 1");
  if (s == &h->opt_epi_async) P2P_REQUIRE(value == 0 || value == 1, "epi_async must be 0 or 1");
  if (s == &h->opt_match_impl) P2P_REQUIRE(value == 0 || value == 1, "match_impl must be 0 or 1");
  if (s == &h->opt_tile_trace) {
    P2P_REQUIRE(value == 0 || value == 1, "tile_trace must be 0 or 1");
    h->traces.clear();
    h->trace_used = 0;
  }
  P2P_REQUIRE(value >= 0, "option values are non-negative");
  *s = value;
  return 0;
}

int p2p_get_option(p2p_handle_t h, const char* key, int* value) {
  P2P_REQUIRE(h != nullptr && key != nullptr && value != nullptr, "null argument");
  if (!strcmp(key, "band_rows")) {  // rows re-computed 3-pass by the last mid-stage call (synchronises)
    *value = 0;
    if (h->last_band_count != nullptr) {
      DeviceGuard g(h->device);
      P2P_CUDA_OK(cudaDeviceSynchronize());
      P2P_CUDA_OK(cudaMemcpy(value, h->last_band_count, sizeof(int), cudaMemcpyDeviceToHost));
    }
    return 0;
  }
  if (!strcmp(key, "frag_epi_launches")) {
    *value = h->frag_epi_launches;
    return 0;
  }
  if (!strcmp(key, "tile_traces")) {
    *value = (int)h->traces.size();
    return 0;
  }
  if (!strcmp(key, "shared_rows")) {  // rows whose conv1 shared a window half in the last mid-stage call (synchronises)
    *value = 0;
    if (h->last_mid_shared && h->share_rows != nullptr) {
      DeviceGuard g(h->device);
      P2P_CUDA_OK(cudaDeviceSynchronize());
      P2P_CUDA_OK(cudaMemcpy(value, h->share_rows, sizeof(int), cudaMemcpyDeviceToHost));
    }
    return 0;
  }
  if (!strcmp(key, "band_rows_total") || !strcmp(key, "band_calls_rows_total")) {
    // running totals since the last read of "band_calls_rows_total" (synchronises): band rows / all mid-stage rows
    *value = 0;
    if (h->band_totals != nullptr) {
      DeviceGuard g(h->device);
      P2P_CUDA_OK(cudaDeviceSynchronize());
      unsigned long long t[2] = {0, 0};
      P2P_CUDA_OK(cudaMemcpy(t, h->band_totals, sizeof(t), cudaMemcpyDeviceToHost));
      const bool rows = !strcmp(key, "band_calls_rows_total");
      *value = (int)(rows ? t[1] : t[0]);
      if (rows) P2P_CUDA_OK(cudaMemset(h->band_totals, 0, sizeof(t)));
    }
    return 0;
  }
  int* s = option_slot(h, key);
  P2P_REQUIRE(s != nullptr, std::string("unknown option ") + key);
  *value = *s;
  return 0;
}

int p2p_launch_count(p2p_handle_t h, long long* count) {
  P2P_REQUIRE(h != nullptr && count != nullptr, "null argument");
  *count = g_launch_count;
  return 0;
}

int p2p_profile_read(p2p_handle_t h, float* ms_by_kind, int* count_by_kind, int nkinds) {
  P2P_ENTER(h);
  P2P_REQUIRE(ms_by_kind && count_by_kind && nkinds >= P2P_PROF_KINDS, "need room for P2P_PROF_KINDS entries");
  for (int i = 0; i < nkinds; ++i) {
    ms_by_kind[i] = 0.f;
    count_by_kind[i] = 0;
  }
  for (auto& e : h->prof) {
    P2P_CUDA_OK(cudaEventSynchronize(e.b));
    float ms = 0.f;
    P2P_CUDA_OK(cudaEventElapsedTime(&ms, e.a, e.b));
    ms_by_kind[e.kind] += ms;
    count_by_kind[e.kind] += 1;
    h->event_pool.push_back(e.a);
    h->event_pool.push_back(e.b);
  }
  h->prof.clear();
  return 0;
}

// -------------------------------------------------------------------------------------------------
// coarse
// -------------------------------------------------------------------------------------------------
static int corr_umma(p2p_handle_s* h, const __half* a_hi, const __half* a_lo, const __half* b_hi, const __half* b_lo,
                     int C, int n1, int n2, int n1pad, int n2pad, int ksize, float* out, uint8_t* code,
                     cudaStream_t st) {
  UmmaGemmParams p;
  memset(&p, 0, sizeof(p));
  const uint64_t ad[5] = {(uint64_t)C, 1, 1, 1, (uint64_t)n1pad};
  const uint64_t as[4] = {(uint64_t)C * 2, (uint64_t)C * 2, (uint64_t)C * 2, (uint64_t)C * 2};
  const uint32_t ab[5] = {64, 1, 1, 1, 128};
  const uint64_t bd[2] = {(uint64_t)C, (uint64_t)n2pad};
  const uint64_t bs[1] = {(uint64_t)C * 2};
  const uint32_t bb[2] = {64, 128};
  int rc;
  if ((rc = make_tmap_fp16(&p.a_main_hi, a_hi, 5, ad, as, ab))) return rc;
  if ((rc = make_tmap_fp16(&p.b_hi, b_hi, 2, bd, bs, bb))) return rc;
  if (h->opt_corr_passes == 3) {
    if ((rc = make_tmap_fp16(&p.a_main_lo, a_lo, 5, ad, as, ab))) return rc;
    if ((rc = make_tmap_fp16(&p.b_lo, b_lo, 2, bd, bs, bb))) return rc;
  }
  p.a_rgb_hi = p.a_main_hi;
  p.a_rgb_lo = p.a_main_hi;
  p.nsteps = C / 64;
  for (int s = 0; s < p.nsteps; ++s) p.steps[s] = KStep{(short)(s * 64), 0, 0, 0, 0, 0, s * 64};
  p.m_tiles = n1pad / 128;
  p.n_tiles = n2pad / 256;
  p.a_units_per_tile = 128;
  p.seg_len = h->opt_seg_len > 0 ? 1 : 0;
  p.epi.c = out;
  p.epi.alpha = 1.f / (kActScale * kActScale);
  if (ksize == 2) {
    p.epi.code = code;
    p.epi.np1 = n1 / 4;
    p.epi.np2 = n2 / 4;
    return launch_umma_gemm(p, EPI_CORR, h->opt_corr_passes, sms(h), st);
  }
  p.epi.ldc = n2;
  p.epi.m_rows = n1;
  p.epi.n_cols = n2;
  return launch_umma_gemm(p, EPI_PLAIN, h->opt_corr_passes, sms(h), st);
}

// The NeighConsensus a coarse-stage or standalone call runs: Patch2Pix's fixed 2-layer stack on the tensor cores
// (nc_umma.cu) or, with option nc_impl 0, on the fp32 kernels (coarse.cu); or NCNet's stack of
// p2p_set_nc_stack_weights (nc_stack.cu).
enum NcKind { kNcUmma, kNcFp32, kNcStack };

// Fails unless the weights of the chosen NeighConsensus are set.
static int pick_nc(const p2p_handle_s* h, bool ncnet, NcKind& kind) {
  if (ncnet)
    P2P_REQUIRE(h->ncs_set, "p2p_set_nc_stack_weights has not been called");
  else
    P2P_REQUIRE(h->nc_set, "p2p_set_ncn_weights has not been called");
  kind = ncnet ? kNcStack : h->opt_nc_impl == 1 ? kNcUmma : kNcFp32;
  return 0;
}

// NeighConsensus scratch.  hidden: fp16 hi/lo [V][64] (nc_umma), fp32 [nA][32][nB] (nc_impl 0) or the stack's lines;
// partial [18][V] f32 and xp only for nc_umma.
struct NcScratch {
  void* hidden = nullptr;
  float* partial = nullptr;
  uint32_t* xp = nullptr;
};

static size_t nc_scratch_bytes(NcKind kind, int hA, int wA, int hB, int wB) {
  const size_t V = (size_t)hA * wA * hB * wB;
  if (kind == kNcUmma) return nc_umma_scratch_bytes(V) + nc_umma_xp_bytes(hA, wA, hB, wB);
  return kind == kNcFp32 ? V * 128 : nc_stack_scratch_bytes(V);
}

static bool carve_nc(Arena& A, NcKind kind, int hA, int wA, int hB, int wB, NcScratch& s) {
  const size_t V = (size_t)hA * wA * hB * wB;
  s.hidden = A.take(kind == kNcStack ? nc_stack_scratch_bytes(V) : V * 128);
  if (kind != kNcUmma) return s.hidden != nullptr;
  s.partial = (float*)A.take(18 * V * 4);
  s.xp = (uint32_t*)A.take(nc_umma_xp_bytes(hA, wA, hB, wB));
  return s.hidden && s.partial && s.xp;
}

// xmax: max |x| (nc_umma, nc_stack).  rowmax / colmax: nc_umma's combine pass also yields the maxima of the
// MutualMatching that follows (may be null).
static int launch_nc(p2p_handle_s* h, NcKind kind, const float* x, int hA, int wA, int hB, int wB, const NcScratch& s,
                     const unsigned int* xmax, float* out, float* rowmax, unsigned int* colmax, cudaStream_t st) {
  if (kind == kNcUmma)
    return launch_neigh_consensus_umma(x, hA, wA, hB, wB, h->ncw, h->nc_b1p, h->nc_b2, xmax, s.xp, (__half*)s.hidden,
                                       s.partial, out, rowmax, colmax, h->opt_nc_l2_mode, sms(h), st);
  if (kind == kNcFp32)
    return launch_neigh_consensus(x, hA, wA, hB, wB, h->nc_w1p, h->nc_b1p, h->nc_w2p, h->nc_b2, (float*)s.hidden, out, st);
  return launch_nc_stack(x, hA, wA, hB, wB, h->ncs, xmax, (__half*)s.hidden, out, sms(h), st);
}

// The coarse stage of one pair: L2-normalise, correlation (+ 4D max-pool for ksize 2), MutualMatching,
// NeighConsensus, MutualMatching.  ncnet: NCNet's stack (fp32 NCHW features, tensor-core correlation only), else
// Patch2Pix's fixed stack.  fmt 1: channels-last fp16 features.
static int coarse_impl(p2p_handle_t h, bool ncnet, const float* feat1, const float* feat2, int fmt, int c, int h1, int w1,
                       int h2, int w2, int ksize, float* corr4d_out, uint8_t* delta_code_out, float* pooled_out,
                       float* ncn_out, void* stream) {
  P2P_ENTER(h);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  NcKind kind;
  int rc = pick_nc(h, ncnet, kind);
  if (rc) return rc;
  P2P_REQUIRE(feat1 && feat2 && corr4d_out, "null tensor pointer");
  P2P_REQUIRE(ksize == 1 || ksize == 2, "ksize must be 1 or 2");
  P2P_REQUIRE(c > 0 && h1 > 0 && w1 > 0 && h2 > 0 && w2 > 0, "empty feature map");
  if (ksize == 2) {
    P2P_REQUIRE(h1 % 2 == 0 && w1 % 2 == 0 && h2 % 2 == 0 && w2 % 2 == 0, "ksize 2 needs even feature sizes");
    P2P_REQUIRE(delta_code_out != nullptr, "delta_code_out is required for ksize 2");
  }
  const bool tc = h->opt_corr_passes > 0;
  if (ncnet) P2P_REQUIRE(tc, "p2p_ncnet_coarse needs the tensor-core correlation (corr_passes 1 or 3)");
  if (tc) P2P_REQUIRE(c % 64 == 0 && c / 64 <= kMaxKSteps, "tensor-core correlation needs C % 64 == 0");
  P2P_REQUIRE(fmt == 0 || tc, "channels-last fp16 features need the tensor-core correlation (corr_passes 1 or 3)");
  const int n1 = h1 * w1, n2 = h2 * w2;
  const int hA = h1 / ksize, wA = w1 / ksize, hB = h2 / ksize, wB = w2 / ksize;
  const int nA = hA * wA, nB = hB * wB;
  const size_t V = (size_t)nA * nB;
  const int n1pad = (int)align_up(n1, 128), n2pad = (int)align_up(n2, 256);
  // pooled, m1, nc [V] f32; the NC scratch; MutualMatching maxima + xmax; the correlation operands (fp16 hi/lo, or fp32)
  const size_t need = 3 * V * 4 + nc_scratch_bytes(kind, hA, wA, hB, wB) + (size_t)(nA + nB) * 4 + 16 +
                      (size_t)(tc ? n1pad + n2pad : n1 + n2) * c * 4 + (1 << 16);
  if ((rc = h->coarse.reserve(need))) return rc;
  Arena& A = h->coarse;
  float* pooled = pooled_out ? pooled_out : (float*)A.take(V * 4);
  float* m1 = (float*)A.take(V * 4);
  float* nc = ncn_out ? ncn_out : (float*)A.take(V * 4);
  NcScratch ns;
  const bool nc_ok = carve_nc(A, kind, hA, wA, hB, wB, ns);
  float* rowmax = (float*)A.take((size_t)nA * 4);
  unsigned int* colmax = (unsigned int*)A.take((size_t)nB * 4 + 16);
  unsigned int* xmax = colmax != nullptr ? colmax + nB : nullptr;
  __half *a_hi = nullptr, *a_lo = nullptr, *b_hi = nullptr, *b_lo = nullptr;   // tensor-core operands
  float *fa = nullptr, *fb = nullptr;                                            // CUDA-core operands (corr_passes 0)
  if (tc) {
    a_hi = (__half*)A.take((size_t)n1pad * c * 2);
    a_lo = (__half*)A.take((size_t)n1pad * c * 2);
    b_hi = (__half*)A.take((size_t)n2pad * c * 2);
    b_lo = (__half*)A.take((size_t)n2pad * c * 2);
  } else {
    fa = (float*)A.take((size_t)n1 * c * 4);
    fb = (float*)A.take((size_t)n2 * c * 4);
  }
  P2P_REQUIRE(pooled && m1 && nc && nc_ok && rowmax && colmax && (tc ? a_hi && a_lo && b_hi && b_lo : fa && fb),
              "scratch carve failed");
  const bool lo = h->opt_corr_passes == 3;
  {
    ProfScope ps(h, P2P_PROF_L2NORM, st);
    if (!tc) {
      if ((rc = launch_l2norm_perm(feat1, fa, c, h1, w1, ksize, st))) return rc;
      rc = launch_l2norm_perm(feat2, fb, c, h2, w2, ksize, st);
    } else if (fmt == 1) {
      rc = launch_l2norm_perm_kmajor_pair_nhwc16(reinterpret_cast<const __half*>(feat1), reinterpret_cast<const __half*>(feat2),
                                                 a_hi, lo ? a_lo : nullptr, b_hi, lo ? b_lo : nullptr, c, h1, w1, h2, w2, ksize, st);
    } else {
      rc = launch_l2norm_perm_kmajor_pair(feat1, feat2, a_hi, lo ? a_lo : nullptr, b_hi, lo ? b_lo : nullptr, c, h1, w1, h2,
                                          w2, ksize, st);
    }
    if (rc) return rc;
  }
  {
    ProfScope ps(h, P2P_PROF_CORR, st);
    rc = tc ? corr_umma(h, a_hi, a_lo, b_hi, b_lo, c, n1, n2, n1pad, n2pad, ksize, pooled, delta_code_out, st)
            : launch_corr_pool_simt(fa, fb, c, n1, n2, ksize, pooled, delta_code_out, st);
    if (rc) return rc;
  }
  {
    ProfScope ps(h, P2P_PROF_MUTUAL, st);
    if ((rc = launch_mutual_matching(pooled, nA, nB, rowmax, colmax, m1, kind == kNcFp32 ? nullptr : xmax, st))) return rc;
  }
  const bool fused_max = kind == kNcUmma;
  {
    ProfScope ps(h, P2P_PROF_NC, st);
    if ((rc = launch_nc(h, kind, m1, hA, wA, hB, wB, ns, xmax, nc, fused_max ? rowmax : nullptr,
                        fused_max ? colmax : nullptr, st)))
      return rc;
  }
  ProfScope ps(h, P2P_PROF_MUTUAL, st);
  if (fused_max) return launch_mutual_apply(nc, nA, nB, rowmax, colmax, corr4d_out, nullptr, st);
  return launch_mutual_matching(nc, nA, nB, rowmax, colmax, corr4d_out, nullptr, st);
}

int p2p_coarse(p2p_handle_t h, const float* feat1, const float* feat2, int c, int h1, int w1, int h2, int w2,
               int ksize, float* corr4d_out, uint8_t* delta_code_out, float* pooled_out, float* ncn_out,
               void* stream) {
  return coarse_impl(h, false, feat1, feat2, 0, c, h1, w1, h2, w2, ksize, corr4d_out, delta_code_out, pooled_out, ncn_out,
                     stream);
}

int p2p_coarse_nhwc16(p2p_handle_t h, const void* feat1_nhwc16, const void* feat2_nhwc16, int c, int h1, int w1, int h2, int w2,
                      int ksize, float* corr4d_out, uint8_t* delta_code_out, float* pooled_out, float* ncn_out,
                      void* stream) {
  return coarse_impl(h, false, reinterpret_cast<const float*>(feat1_nhwc16), reinterpret_cast<const float*>(feat2_nhwc16), 1,
                     c, h1, w1, h2, w2, ksize, corr4d_out, delta_code_out, pooled_out, ncn_out, stream);
}

int p2p_ncnet_coarse(p2p_handle_t h, const float* feat1, const float* feat2, int c, int h1, int w1, int h2, int w2, int ksize,
                     float* corr4d_out, uint8_t* delta_code_out, void* stream) {
  return coarse_impl(h, true, feat1, feat2, 0, c, h1, w1, h2, w2, ksize, corr4d_out, delta_code_out, nullptr, nullptr,
                     stream);
}

int p2p_delta_unpack(p2p_handle_t h, const uint8_t* code, long long n, int ksize, int64_t* di, int64_t* dj,
                     int64_t* dk, int64_t* dl, void* stream) {
  P2P_ENTER(h);
  P2P_REQUIRE(code && di && dj && dk && dl && n >= 0 && ksize >= 1 && ksize <= 3, "bad argument");
  if (n == 0) return 0;
  return launch_delta_unpack(code, (size_t)n, ksize, (long long*)di, (long long*)dj, (long long*)dk, (long long*)dl,
                             reinterpret_cast<cudaStream_t>(stream));
}

int p2p_delta_pack(p2p_handle_t h, const int64_t* di, const int64_t* dj, const int64_t* dk, const int64_t* dl,
                   long long n, int ksize, uint8_t* code, void* stream) {
  P2P_ENTER(h);
  P2P_REQUIRE(code && di && dj && dk && dl && n >= 0 && ksize >= 1 && ksize <= 3, "bad argument");
  if (n == 0) return 0;
  return launch_delta_pack((const long long*)di, (const long long*)dj, (const long long*)dk, (const long long*)dl,
                           (size_t)n, ksize, code, reinterpret_cast<cudaStream_t>(stream));
}

int p2p_mutual_matching(p2p_handle_t h, const float* in, int nA, int nB, float* out, void* stream) {
  P2P_ENTER(h);
  P2P_REQUIRE(in && out && nA > 0 && nB > 0, "bad argument");
  int rc = h->misc.reserve((size_t)(nA + nB) * 4 + 4096);
  if (rc) return rc;
  float* rowmax = (float*)h->misc.take((size_t)nA * 4);
  unsigned int* colmax = (unsigned int*)h->misc.take((size_t)nB * 4);
  return launch_mutual_matching(in, nA, nB, rowmax, colmax, out, nullptr, reinterpret_cast<cudaStream_t>(stream));
}

// NeighConsensus alone on [hA, wA, hB, wB]: Patch2Pix's fixed stack (p2p_neigh_consensus) or NCNet's (p2p_nc_stack).
static int nc_alone(p2p_handle_t h, bool ncnet, const float* in, int hA, int wA, int hB, int wB, float* out, void* stream) {
  P2P_ENTER(h);
  NcKind kind;
  int rc = pick_nc(h, ncnet, kind);
  if (rc) return rc;
  P2P_REQUIRE(in && out && hA > 0 && wA > 0 && hB > 0 && wB > 0, "bad argument");
  if ((rc = h->misc.reserve(nc_scratch_bytes(kind, hA, wA, hB, wB) + 8192))) return rc;
  NcScratch ns;
  const bool nc_ok = carve_nc(h->misc, kind, hA, wA, hB, wB, ns);
  unsigned int* xmax = (unsigned int*)h->misc.take(16);
  P2P_REQUIRE(nc_ok && xmax, "scratch carve failed");
  if (!ncnet) {
    h->dbg_nc[0] = ns.hidden; h->dbg_nc[1] = ns.partial; h->dbg_nc[2] = ns.xp; h->dbg_nc[3] = xmax;
  }
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  ProfScope ps(h, P2P_PROF_NC, st);
  if (kind != kNcFp32 && (rc = launch_absmax(in, (size_t)hA * wA * hB * wB, xmax, st))) return rc;
  return launch_nc(h, kind, in, hA, wA, hB, wB, ns, xmax, out, nullptr, nullptr, st);
}

int p2p_neigh_consensus(p2p_handle_t h, const float* in, int hA, int wA, int hB, int wB, float* out, void* stream) {
  return nc_alone(h, false, in, hA, wA, hB, wB, out, stream);
}

int p2p_nc_stack(p2p_handle_t h, const float* in, int hA, int wA, int hB, int wB, float* out, void* stream) {
  return nc_alone(h, true, in, hA, wA, hB, wB, out, stream);
}

// Development hook (not part of include/p2p_b200.h): copies `bytes` of an intermediate of the last
// p2p_neigh_consensus call to the host -- which = 0 hidden [V][64] fp16, 1 partial [18][V] f32, 2 xp (padded hi|lo
// words), 3 xmax word.  Under nc_impl 0 only 0 (hidden, fp32 [nA][32][nB]) and 3 are set.
P2P_API int p2p_debug_nc_scratch(p2p_handle_t h, int which, void* host_dst, size_t bytes) {
  P2P_ENTER(h);
  P2P_REQUIRE(which >= 0 && which < 4 && host_dst != nullptr && h->dbg_nc[which] != nullptr, "bad argument");
  P2P_CUDA_OK(cudaDeviceSynchronize());
  P2P_CUDA_OK(cudaMemcpy(host_dst, h->dbg_nc[which], bytes, cudaMemcpyDeviceToHost));
  return 0;
}

int p2p_proposals(p2p_handle_t h, const float* corr4d, const uint8_t* delta_code, int hA, int wA, int hB, int wB,
                  int ksize, int upsample, int center, int do_softmax, int64_t* matches_out, float* scores_out,
                  void* stream) {
  P2P_ENTER(h);
  P2P_REQUIRE(corr4d && matches_out && scores_out, "null tensor pointer");
  P2P_REQUIRE(hA > 0 && wA > 0 && hB > 0 && wB > 0 && ksize >= 1 && ksize <= 3 && upsample > 0, "bad dims");
  P2P_REQUIRE(ksize == 1 || delta_code != nullptr, "delta_code is required for ksize > 1");
  ProfScope ps(h, P2P_PROF_PROPOSALS, reinterpret_cast<cudaStream_t>(stream));
  return launch_proposals(corr4d, ksize > 1 ? delta_code : nullptr, hA, wA, hB, wB, ksize, upsample, center,
                          do_softmax, (long long*)matches_out, scores_out, reinterpret_cast<cudaStream_t>(stream));
}

int p2p_proposals_topk(p2p_handle_t h, const float* corr4d, const uint8_t* delta_code, int b, int hA, int wA, int hB,
                       int wB, int topk, int ksize, int do_softmax, int invert, int64_t* jA_out, int64_t* iA_out,
                       int64_t* jB_out, int64_t* iB_out, float* scores_out, void* stream) {
  P2P_ENTER(h);
  P2P_REQUIRE(corr4d && jA_out && iA_out && jB_out && iB_out && scores_out, "null tensor pointer");
  P2P_REQUIRE(b > 0 && b <= 65535 && hA > 0 && wA > 0 && hB > 0 && wB > 0 && ksize >= 1 && ksize <= 3, "bad dims");
  P2P_REQUIRE((long long)hA * wA <= INT32_MAX && (long long)hB * wB <= INT32_MAX, "bad dims");
  const int n_slice = invert ? hB * wB : hA * wA;
  P2P_REQUIRE(n_slice <= kTopkMaxSlice, "slice longer than 32768 cells");
  P2P_REQUIRE(topk >= 1 && topk <= n_slice, "topk must be in 1..slice length");
  P2P_REQUIRE(ksize == 1 || delta_code != nullptr, "delta_code is required for ksize > 1");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  ProfScope ps(h, P2P_PROF_PROPOSALS, st);
  return launch_corr_topk(corr4d, ksize > 1 ? delta_code : nullptr, b, hA, wA, hB, wB, topk, ksize, do_softmax != 0,
                          invert != 0, (long long*)jA_out, (long long*)iA_out, (long long*)jB_out, (long long*)iB_out,
                          scores_out, st);
}

int p2p_unique_rows(p2p_handle_t h, const int64_t* rows, int n, int mutual, const float* scores, float thres,
                    int32_t* ids_out, int32_t* count_out, void* stream) {
  P2P_ENTER(h);
  P2P_REQUIRE(rows && ids_out && count_out, "null tensor pointer");
  unsigned char* scratch = nullptr;
  const size_t sb = unique_rows_scratch_bytes(n);
  if (sb > 0) {   // candidate lists beyond 16384 rows sort in global scratch (same kernel, same result)
    int rc = h->uniq.reserve(sb + 4096);
    if (rc) return rc;
    scratch = (unsigned char*)h->uniq.take(sb);
  }
  if (h->uniq_rank == nullptr && h->opt_unique_impl == 1) {     // zeroed once; the kernel leaves it zeroed
    P2P_CUDA_OK(cudaMalloc(&h->uniq_rank, unique_rank_scratch_bytes()));
    P2P_CUDA_OK(cudaMemset(h->uniq_rank, 0, unique_rank_scratch_bytes()));
  }
  ProfScope ps(h, P2P_PROF_PROPOSALS, reinterpret_cast<cudaStream_t>(stream));
  return launch_unique_rows((const long long*)rows, n, mutual, scores, thres, ids_out, count_out, scratch,
                            h->opt_unique_impl == 1 ? h->uniq_rank : nullptr, reinterpret_cast<cudaStream_t>(stream));
}

int p2p_select_anchor(p2p_handle_t h, const int64_t* rows, const float* scores, const int32_t* ids, const int32_t* sel,
                      int m, int panc, int pshift, int64_t* matches_out, float* scores_out, int64_t* anchors_out,
                      void* stream) {
  P2P_ENTER(h);
  P2P_REQUIRE(m >= 0 && rows != nullptr, "bad argument");
  P2P_REQUIRE(panc == 1 || panc == 8, "panc must be 1 or 8 (networks/patch2pix.py:377-402)");
  P2P_REQUIRE(scores_out == nullptr || scores != nullptr, "scores_out needs scores");
  P2P_REQUIRE(panc == 1 || anchors_out != nullptr, "anchors_out is required for panc 8");
  ProfScope ps(h, P2P_PROF_PROPOSALS, reinterpret_cast<cudaStream_t>(stream));
  return launch_select_anchor((const long long*)rows, scores, ids, sel, m, panc, pshift, (long long*)matches_out,
                              scores_out, (long long*)anchors_out, reinterpret_cast<cudaStream_t>(stream));
}

// -------------------------------------------------------------------------------------------------
// refine
// -------------------------------------------------------------------------------------------------
static int refine_prepare_impl(p2p_handle_t h, const float* const* feats1, const float* const* feats2, int fmt, int H1, int W1,
                               int H2, int W2, void* stream) {
  P2P_ENTER(h);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  P2P_REQUIRE(feats1 && feats2, "null feature list");
  for (int l = 0; l < 4; ++l) P2P_REQUIRE(feats1[l] && feats2[l], "null feature level");
  // below 8 px the reference's level-3 clamp bound W // 8 - 1 is -1 and its index wraps around
  P2P_REQUIRE(H1 >= 8 && W1 >= 8 && H2 >= 8 && W2 >= 8, "image sizes must be at least 8 x 8");
  const int Hs[2] = {H1, H2}, Ws[2] = {W1, W2};
  size_t need = 1 << 16;
  for (int s = 0; s < 2; ++s) {
    const size_t px = (size_t)Hs[s] * Ws[s];
    need += (px / 4 * 64 + px / 16 * 64 + px / 64 * 128) * 6 + (px + px / 4 + px / 16 + px / 64) * 4 + 32768;
  }
  const bool want_map = h->opt_fuse_gather == 3;
  if (want_map)
    for (int s = 0; s < 2; ++s) need += (size_t)(Hs[s] + 2 * kMapPad) * map_pitch(Ws[s]) * (512 + 8) + 4096;
  int rc = h->feat.reserve(need);
  if (rc) return rc;
  const int chans[3] = {64, 64, 128};
  for (int s = 0; s < 2; ++s) {
    PairFeatures& pf = h->pf[s];
    for (int l = 0; l < 4; ++l) {
      const int ds = 1 << l;
      pf.nsq[l] = (float*)h->feat.take((size_t)(Hs[s] / ds) * (Ws[s] / ds) * 4);   // the floor-sized crop
      P2P_REQUIRE(pf.nsq[l] != nullptr, "scratch carve failed");
    }
    for (int l = 0; l < 3; ++l) {
      const int ds = 2 << l;
      pf.nhwc[l] = (float*)h->feat.take((size_t)(Hs[s] / ds) * (Ws[s] / ds) * chans[l] * 4);
      pf.nhwc16[l] = (__half*)h->feat.take((size_t)(Hs[s] / ds) * (Ws[s] / ds) * chans[l] * 2);
      P2P_REQUIRE(pf.nhwc[l] != nullptr && pf.nhwc16[l] != nullptr, "scratch carve failed");
    }
    pf.wmap = pf.rgbn = nullptr;
    if (want_map) {
      const size_t pxp = (size_t)(Hs[s] + 2 * kMapPad) * map_pitch(Ws[s]);
      pf.wmap = (__half*)h->feat.take(pxp * 512);
      pf.rgbn = (__half*)h->feat.take(pxp * 8);
      P2P_REQUIRE(pf.wmap != nullptr && pf.rgbn != nullptr, "scratch carve failed");
    }
  }
  {
    ProfScope ps(h, P2P_PROF_PREP, st);
    if ((rc = launch_feature_prep_pair(feats1, feats2, Hs, Ws, h->pf, fmt, st))) return rc;
    if (want_map && (rc = launch_window_map(h->pf, st))) return rc;
  }
  h->prepared = true;
  return 0;
}

int p2p_refine_prepare(p2p_handle_t h, const float* const* feats1, const float* const* feats2, int H1, int W1,
                       int H2, int W2, void* stream) {
  return refine_prepare_impl(h, feats1, feats2, 0, H1, W1, H2, W2, stream);
}

int p2p_refine_prepare_nhwc16(p2p_handle_t h, const void* const* feats1, const void* const* feats2, int H1, int W1,
                              int H2, int W2, void* stream) {
  return refine_prepare_impl(h, reinterpret_cast<const float* const*>(feats1), reinterpret_cast<const float* const*>(feats2), 1,
                             H1, W1, H2, W2, stream);
}

namespace {

struct RefineBuffers {
  __half *p_hi, *p_lo, *r_hi, *r_lo, *y_hi, *y_lo;
  __half *q_hi, *q_lo, *h1_hi, *h1_lo, *h2_hi, *h2_lo;   // tensor-core FC operands, rows padded to 128
  float *pooled, *raw;
  int *rowmap, *d_count;
  int *sh_prefix, *sh_cont, *sh_unsh, *sh_cnt;   // launch_window_share_classify's lists and counts
  float* part;                                    // share_windows: fp32 partial sums of the prefix launch
  __half* r_unsh;                                 // share_windows: rgb im2col rows of the unshared rows
  int npad;
};

// The 36 conv1 k-steps of image si's window map (chunks 4 si .. 4 si + 3 of every tap), in tap-major order.
int image_steps(const Regressor& R, int si, KStep* out) {
  int k = 0;
  for (int s = 0; s < 72; ++s)
    if ((R.steps1[s].c0 >> 6) >> 2 == si) out[k++] = R.steps1[s];
  return k;
}

// gather -> conv1 -> conv2 -> fc/parse for the rows selected by (rowmap, d_count) [all rows if null]
int run_regressor(p2p_handle_s* h, Regressor& R, int which, int passes, const RefineBuffers& B, const void* matches_in,
                  int is_float, int n, const int* rowmap, const int* d_count, float* matches_out, float* probs_out,
                  float* raw_out, cudaStream_t st) {
  const bool lo = passes == 3;
  const int kb = rowmap != nullptr ? P2P_PROF_GATHER_BAND : (which == 0 ? P2P_PROF_GATHER_MID : P2P_PROF_GATHER_FINE);
  int rc;
  const bool mapped = passes == 1 && rowmap == nullptr && h->opt_fuse_gather == 3 && h->opt_gemm_impl == 0;
  const bool fused = passes == 1 && rowmap == nullptr && h->opt_fuse_gather && h->opt_gemm_impl == 0 && !mapped;
  if (mapped) P2P_REQUIRE(h->pf[0].wmap != nullptr && h->pf[1].wmap != nullptr,
                          "fuse_gather = 3 needs p2p_refine_prepare to have run with the same option");
  // Mid-stage anchor groups (shift_to_anchors): rows 8g..8g+3 share image 2's window, rows 8g+4..8g+7 image 1's.  conv1
  // is linear in its input channels, so a shared window's 36 k-steps run once per half-group (prefix launch) and each
  // row adds that partial sum to its own 37 (continuation launch); the other rows run all 73 k-steps as before.
  const bool share = mapped && which == 0 && h->opt_share_windows;
  if (which == 0 && rowmap == nullptr) h->last_mid_shared = share;
  if (!fused && !mapped) {
    ProfScope ps(h, kb, st);
    if ((rc = launch_patch_gather(h->pf[0], h->pf[1], matches_in, is_float, n, B.p_hi, lo ? B.p_lo : nullptr, B.r_hi,
                                  lo ? B.r_lo : nullptr, rowmap, d_count, st)))
      return rc;
  }
  if (h->opt_gemm_impl == 1) {
    P2P_REQUIRE(rowmap == nullptr, "the CUDA-core checker GEMM does not support row subsets");
    GemmOperands g1 = {B.p_hi, B.p_lo, B.r_hi, B.r_lo, R.w1_hi, R.w1_lo, 4, kConv1Steps * 64, n, passes, R.d_steps1, kConv1Steps};
    ConvEpilogue e1 = {R.scale1, R.bias1, 0, R.y_scale, B.y_hi, lo ? B.y_lo : nullptr, nullptr};
    {
      ProfScope ps(h, kb + 1, st);
      if ((rc = launch_conv_gemm_simt(g1, e1, st))) return rc;
    }
    ProfScope ps(h, kb + 2, st);
    GemmOperands g2 = {B.y_hi, B.y_lo, nullptr, nullptr, R.w2_hi, R.w2_lo, 1, kConv2Steps * 64, n, passes, R.d_steps2, kConv2Steps};
    ConvEpilogue e2 = {R.scale2, R.bias2, 1, 1.f, nullptr, nullptr, B.pooled};
    if ((rc = launch_conv_gemm_simt(g2, e2, st))) return rc;
  } else {
    UmmaGemmParams p;
    memset(&p, 0, sizeof(p));
    const uint32_t abox[5] = {64, 8, 8, 1, 2};
    const uint32_t bbox[2] = {64, 128};
    const uint64_t npad = (uint64_t)B.npad;
    {  // conv1
      const uint64_t ad[5] = {512, 8, 8, 4, npad};
      const uint64_t as[4] = {1024, 8192, 65536, 262144};
      const uint64_t rd[5] = {64, 8, 8, 1, npad};
      const uint64_t rs[4] = {128, 1024, 8192, 8192};
      const uint64_t bd[2] = {(uint64_t)kConv1Steps * 64, 512};
      const uint64_t bs[1] = {(uint64_t)kConv1Steps * 64 * 2};
      if ((rc = make_tmap_fp16(&p.a_main_hi, B.p_hi, 5, ad, as, abox))) return rc;
      if ((rc = make_tmap_fp16(&p.a_rgb_hi, B.r_hi, 5, rd, rs, abox))) return rc;
      if ((rc = make_tmap_fp16(&p.b_hi, R.w1_hi, 2, bd, bs, bbox))) return rc;
      if ((rc = make_tmap_fp16(&p.a_main_lo, lo ? B.p_lo : B.p_hi, 5, ad, as, abox))) return rc;
      if ((rc = make_tmap_fp16(&p.a_rgb_lo, lo ? B.r_lo : B.r_hi, 5, rd, rs, abox))) return rc;
      if ((rc = make_tmap_fp16(&p.b_lo, R.w1_lo, 2, bd, bs, bbox))) return rc;
      p.nsteps = kConv1Steps;
      memcpy(p.steps, R.steps1, sizeof(R.steps1));
      p.m_tiles = (n + 1) / 2;
      p.n_tiles = 2;
      p.a_units_per_tile = 2;
      p.seg_len = lo ? h->opt_seg_len : 0;
      p.d_units = d_count;
      p.epi.scale = R.scale1;
      p.epi.bias = R.bias1;
      p.epi.y_scale = R.y_scale;
      p.epi.y_hi = B.y_hi;
      p.epi.y_lo = lo ? B.y_lo : nullptr;
      p.epi.pooled = B.pooled;       // conv1's epilogue zeroes the max-pool accumulator conv2 merges into
      p.epi.n_patches = n;
      // 1-pass: conv1 and conv2 run on 256-wide tiles, which the fragment epilogues serve
      p.frag_epi = !lo && !fused && h->opt_epi_async;
      if (p.frag_epi) {
        const uint64_t yd[3] = {512, 64, npad};
        const uint64_t ys[2] = {1024, 65536};
        const uint32_t yb[3] = {64, 64, 1};
        if ((rc = make_tmap_fp16(&p.y_store, B.y_hi, 3, yd, ys, yb))) return rc;
      }
      if (fused) {
        for (int s2 = 0; s2 < 2; ++s2) {
          p.fg.img[s2] = h->pf[s2].img;
          for (int l = 0; l < 3; ++l) p.fg.nhwc16[s2][l] = h->pf[s2].nhwc16[l];
          for (int l = 0; l < 4; ++l) p.fg.nsq[s2][l] = h->pf[s2].nsq[l];
          p.fg.H[s2] = h->pf[s2].H;
          p.fg.W[s2] = h->pf[s2].W;
        }
        p.fg.matches = matches_in;
        p.fg.is_float = is_float;
      }
      if (mapped) {
        for (int s2 = 0; s2 < 2; ++s2) {
          const uint64_t Wp = (uint64_t)map_pitch(h->pf[s2].W), Hp = (uint64_t)h->pf[s2].H + 2 * kMapPad;
          const uint64_t md[3] = {256, Wp, Hp};
          const uint64_t ms[2] = {512, Wp * 512};
          const uint32_t mb[3] = {64, 16, 16};       // 8 elements at traversal stride 2 (box = N * stride)
          const uint32_t me[3] = {1, 2, 2};
          if ((rc = make_tmap_fp16(&p.wm.map[s2], h->pf[s2].wmap, 3, md, ms, mb, me))) return rc;
          p.wm.rgbn[s2] = h->pf[s2].rgbn;
          p.wm.H[s2] = h->pf[s2].H;
          p.wm.W[s2] = h->pf[s2].W;
        }
        p.wm.matches = matches_in;
        p.wm.is_float = is_float;
        // the rgb k-step's A operand (r_hi, read through a_rgb_hi); the main k-steps read the window maps directly.
        // Shared: the rows are classified first; r_hi holds the continuation order, r_unsh the unshared rows' order.
        ProfScope ps(h, kb, st);
        if (share) {
          P2P_REQUIRE(B.part != nullptr && B.r_unsh != nullptr, "share_windows: buffers not carved");
          if ((rc = launch_window_share_classify(p.wm, n, B.sh_prefix, B.sh_cont, B.sh_unsh, B.sh_cnt, h->share_rows, st)))
            return rc;
          if ((rc = launch_window_rgb(p.wm, n, B.npad, B.r_hi, st, B.sh_cont, B.sh_cnt + 3))) return rc;
          if ((rc = launch_window_rgb(p.wm, n, B.npad, B.r_unsh, st, B.sh_unsh, B.sh_cnt + 6))) return rc;
        } else if ((rc = launch_window_rgb(p.wm, n, B.npad, B.r_hi, st))) {
          return rc;
        }
      }
      ProfScope ps(h, kb + 1, st);
      const int amode = mapped ? AMODE_WINDOW : (fused ? AMODE_GATHER : AMODE_TMA);
      const int tg = (rowmap != nullptr ? 2 : which) * 8;   // tile_trace tag: stage * 8 + launch kind
      if (share) {
        float* part = B.part;   // fp32 partial sums, [prefix slot][2][64][256]
        KStep img[2][36];
        image_steps(R, 0, img[0]);
        image_steps(R, 1, img[1]);
        UmmaGemmParams q = p;
        // prefix: A half-groups (image 2's steps), then B half-groups (image 1's)
        memcpy(q.steps, img[1], sizeof(img[1]));
        memcpy(q.steps + 36, img[0], sizeof(img[0]));
        q.nsteps = 36;
        q.m_tiles = (n / 4 + 3) / 2;
        q.d_units = B.sh_cnt;
        q.ws = WindowShare{B.sh_prefix, B.sh_cnt + 1, 36, part, nullptr};
        if ((rc = set_trace(h, q, tg + 1, st))) return rc;
        if ((rc = launch_umma_gemm(q, EPI_CONV1, passes, sms(h), st, amode))) return rc;
        // continuation: A rows run image 1's steps + rgb, B rows image 2's + rgb
        memcpy(q.steps, img[0], sizeof(img[0]));
        q.steps[36] = R.steps1[72];
        memcpy(q.steps + 37, img[1], sizeof(img[1]));
        q.steps[73] = R.steps1[72];
        q.nsteps = 37;
        q.m_tiles = (n + 1) / 2;
        q.d_units = B.sh_cnt + 3;
        q.ws = WindowShare{B.sh_cont, B.sh_cnt + 4, 37, nullptr, part};
        if ((rc = set_trace(h, q, tg + 2, st))) return rc;
        if ((rc = launch_umma_gemm(q, EPI_CONV1, passes, sms(h), st, amode))) return rc;
        // unshared rows: all 73 steps, exactly as without sharing
        q = p;
        if ((rc = make_tmap_fp16(&q.a_rgb_hi, B.r_unsh, 5, rd, rs, abox))) return rc;
        q.d_units = B.sh_cnt + 6;
        q.ws = WindowShare{B.sh_unsh, nullptr, 0, nullptr, nullptr};
        if ((rc = set_trace(h, q, tg + 3, st))) return rc;
        if ((rc = launch_umma_gemm(q, EPI_CONV1, passes, sms(h), st, amode))) return rc;
      } else {
        if ((rc = set_trace(h, p, tg, st))) return rc;
        if ((rc = launch_umma_gemm(p, EPI_CONV1, passes, sms(h), st, amode))) return rc;
      }
      h->frag_epi_launches += p.frag_epi ? (share ? 3 : 1) : 0;
    }
    {  // conv2
      const uint64_t ad[5] = {512, 8, 8, 1, npad};
      const uint64_t as[4] = {1024, 8192, 65536, 65536};
      const uint64_t bd[2] = {(uint64_t)kConv2Steps * 64, 512};
      const uint64_t bs[1] = {(uint64_t)kConv2Steps * 64 * 2};
      if ((rc = make_tmap_fp16(&p.a_main_hi, B.y_hi, 5, ad, as, abox))) return rc;
      if ((rc = make_tmap_fp16(&p.a_main_lo, lo ? B.y_lo : B.y_hi, 5, ad, as, abox))) return rc;
      if ((rc = make_tmap_fp16(&p.b_hi, R.w2_hi, 2, bd, bs, bbox))) return rc;
      if ((rc = make_tmap_fp16(&p.b_lo, R.w2_lo, 2, bd, bs, bbox))) return rc;
      p.a_rgb_hi = p.a_main_hi;
      p.a_rgb_lo = p.a_main_lo;
      p.nsteps = kConv2Steps;
      memcpy(p.steps, R.steps2, sizeof(R.steps2));
      p.epi.scale = R.scale2;
      p.epi.bias = R.bias2;
      p.epi.pooled = B.pooled;
      if ((rc = set_trace(h, p, (rowmap != nullptr ? 2 : which) * 8 + 4, st))) return rc;
      ProfScope ps(h, kb + 2, st);
      if ((rc = launch_umma_gemm(p, EPI_CONV2, passes, sms(h), st))) return rc;
      h->frag_epi_launches += p.frag_epi;
    }
  }
  ProfScope ps(h, kb + 3, st);
  if (h->opt_fc_impl == 0 || h->opt_gemm_impl == 1)
    return launch_fc_parse(B.pooled, R.fc, matches_in, is_float, n, h->pf[0].W, h->pf[0].H, h->pf[1].W, h->pf[1].H,
                           matches_out, probs_out, raw_out, rowmap, d_count, st);
  // tensor-core FC: split -> Linear(512,512)+BN+ReLU -> Linear(512,256)+BN+ReLU (3-pass, segmented) -> Linear(256,5)+parse
  if ((rc = launch_pooled_split(B.pooled, n, R.fc_scale[0], B.q_hi, B.q_lo, d_count, st))) return rc;
  const uint64_t m128 = align_up(n, 128);
  const uint32_t abx[5] = {64, 1, 1, 1, 128};
  const uint32_t bbx[2] = {64, 128};
  for (int layer = 0; layer < 2; ++layer) {
    UmmaGemmParams p;
    memset(&p, 0, sizeof(p));
    const int nout = layer == 0 ? 512 : 256;
    const uint64_t ad[5] = {512, 1, 1, 1, m128};
    const uint64_t as[4] = {1024, 1024, 1024, 1024};
    const uint64_t bd[2] = {512, (uint64_t)nout};
    const uint64_t bs[1] = {1024};
    const __half* a_hi = layer == 0 ? B.q_hi : B.h1_hi;
    const __half* a_lo = layer == 0 ? B.q_lo : B.h1_lo;
    if ((rc = make_tmap_fp16(&p.a_main_hi, a_hi, 5, ad, as, abx))) return rc;
    if ((rc = make_tmap_fp16(&p.a_main_lo, a_lo, 5, ad, as, abx))) return rc;
    if ((rc = make_tmap_fp16(&p.b_hi, layer == 0 ? R.f1_hi : R.f2_hi, 2, bd, bs, bbx))) return rc;
    if ((rc = make_tmap_fp16(&p.b_lo, layer == 0 ? R.f1_lo : R.f2_lo, 2, bd, bs, bbx))) return rc;
    p.a_rgb_hi = p.a_main_hi;
    p.a_rgb_lo = p.a_main_lo;
    p.nsteps = 8;
    for (int s2 = 0; s2 < 8; ++s2) p.steps[s2] = KStep{(short)(s2 * 64), 0, 0, 0, 0, 0, s2 * 64};
    p.m_tiles = (int)(m128 / 128);
    p.n_tiles = nout / 256;
    p.a_units_per_tile = 128;
    p.seg_len = 2;
    p.d_units = d_count;
    p.epi.scale = layer == 0 ? R.fa1 : R.fa2;
    p.epi.bias = layer == 0 ? R.fc.b1 : R.fc.b2;
    p.epi.y_scale = R.fc_scale[layer + 1];
    p.epi.y_hi = layer == 0 ? B.h1_hi : B.h2_hi;
    p.epi.y_lo = layer == 0 ? B.h1_lo : B.h2_lo;
    p.epi.ldc = nout;
    p.epi.n_patches = n;
    if ((rc = launch_umma_gemm(p, EPI_FC, 3, sms(h), st))) return rc;
  }
  return launch_fc3_parse(B.h2_hi, B.h2_lo, 1.f / R.fc_scale[2], R.fc.w3t, R.fc.b3, matches_in, is_float, n, h->pf[0].W, h->pf[0].H,
                          h->pf[1].W, h->pf[1].H, matches_out, probs_out, raw_out, rowmap, d_count, st);
}

}  // namespace

int p2p_refine(p2p_handle_t h, int which, const void* matches_in, int is_float, int n, float* matches_out,
               float* probs_out, void* stream) {
  P2P_ENTER(h);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  P2P_REQUIRE(which == 0 || which == 1, "which must be 0 (mid) or 1 (fine)");
  P2P_REQUIRE(h->reg[which].set, "p2p_set_regressor_weights has not been called for this regressor");
  P2P_REQUIRE(h->prepared, "p2p_refine_prepare has not been called");
  P2P_REQUIRE(n >= 0, "negative match count");
  if (n == 0) return 0;
  P2P_REQUIRE(matches_in && matches_out && probs_out, "null tensor pointer");
  Regressor& R = h->reg[which];
  const int passes = which == 0 ? h->opt_mid_passes : h->opt_fine_passes;
  // Risk band (mid stage only): 1-pass for every row, fp32-grade 3-pass re-computation only for the
  // rows whose coordinates sit within mid_band/1000 px of an integer (trunc() must match the reference).
  const bool band = which == 0 && passes == 3 && h->opt_mid_band > 0 && h->opt_gemm_impl == 0;
  const int npad = (int)align_up(n, 2);
  const size_t pbytes = (size_t)npad * kPatchPos * kMainCh * 2, rbytes = (size_t)npad * 4096 * 2,
               ybytes = (size_t)npad * 64 * 512 * 2, qbytes = (size_t)npad * 512 * 4;
  const size_t n128 = align_up(n, 128);
  const size_t shbytes = ((size_t)n * 2 + n / 4 + 2 + 8) * 4;
  // share_windows: partial sums (one 128 KB unit per prefix slot, at most n / 4 + 1 slots) and the unshared rows' rgb
  const bool share_bufs = which == 0 && h->opt_share_windows;
  const size_t partbytes = share_bufs ? ((size_t)n / 4 + 2) * 64 * 512 * 4 : 0, runshbytes = share_bufs ? rbytes : 0;
  int rc = h->refine.reserve(2 * (pbytes + rbytes + ybytes) + qbytes + (size_t)n * 24 + n128 * (512 + 512 + 256) * 4 +
                             shbytes + partbytes + runshbytes + (1 << 16));
  if (rc) return rc;
  Arena& A = h->refine;
  RefineBuffers B;
  B.npad = npad;
  B.p_hi = (__half*)A.take(pbytes);
  B.p_lo = (__half*)A.take(pbytes);
  B.r_hi = (__half*)A.take(rbytes);
  B.r_lo = (__half*)A.take(rbytes);
  B.y_hi = (__half*)A.take(ybytes);
  B.y_lo = (__half*)A.take(ybytes);
  B.pooled = (float*)A.take(qbytes);
  B.q_hi = (__half*)A.take(n128 * 512 * 2);
  B.q_lo = (__half*)A.take(n128 * 512 * 2);
  B.h1_hi = (__half*)A.take(n128 * 512 * 2);
  B.h1_lo = (__half*)A.take(n128 * 512 * 2);
  B.h2_hi = (__half*)A.take(n128 * 256 * 2);
  B.h2_lo = (__half*)A.take(n128 * 256 * 2);
  B.raw = (float*)A.take((size_t)n * 5 * 4);
  B.rowmap = (int*)A.take((size_t)n * 4 + 16);
  B.sh_cnt = (int*)A.take(shbytes);
  B.part = share_bufs ? (float*)A.take(partbytes) : nullptr;
  B.r_unsh = share_bufs ? (__half*)A.take(runshbytes) : nullptr;
  P2P_REQUIRE(B.p_hi && B.p_lo && B.r_hi && B.r_lo && B.y_hi && B.y_lo && B.pooled && B.raw && B.rowmap && B.q_hi &&
                  B.q_lo && B.h1_hi && B.h1_lo && B.h2_hi && B.h2_lo && B.sh_cnt &&
                  (!share_bufs || (B.part && B.r_unsh)),
              "scratch carve failed");
  B.sh_prefix = B.sh_cnt + 8;
  B.sh_cont = B.sh_prefix + n / 4 + 2;
  B.sh_unsh = B.sh_cont + n;
  B.d_count = B.rowmap + n;
  if (which == 0) h->last_band_count = band ? B.d_count : nullptr;
  auto& T = h->tap;
  T.y_hi = B.y_hi;
  T.y_lo = B.y_lo;
  T.pooled = B.pooled;
  T.h1_hi = B.h1_hi;
  T.h1_lo = B.h1_lo;
  T.h2_hi = B.h2_hi;
  T.h2_lo = B.h2_lo;
  T.raw = B.raw;
  T.rowmap = band ? B.rowmap : nullptr;
  T.d_count = band ? B.d_count : nullptr;
  T.n = n;
  T.passes = passes;
  T.fc_tc = h->opt_fc_impl != 0 && h->opt_gemm_impl == 0;
  T.scales[0] = R.y_scale;
  for (int i = 0; i < 3; ++i) T.scales[i + 1] = R.fc_scale[i];
  if (!band)
    return run_regressor(h, R, which, passes, B, matches_in, is_float, n, nullptr, nullptr, matches_out, probs_out,
                         B.raw, st);
  if ((rc = run_regressor(h, R, which, 1, B, matches_in, is_float, n, nullptr, nullptr, matches_out, probs_out, B.raw,
                          st)))
    return rc;
  {
    ProfScope ps(h, P2P_PROF_FLAG, st);
    if ((rc = launch_flag_risky(matches_in, is_float, B.raw, n, h->opt_mid_band * 1e-3f, 0.02f, h->pf[0].W, h->pf[0].H,
                                h->pf[1].W, h->pf[1].H, B.rowmap, B.d_count, h->band_totals, st)))
      return rc;
  }
  return run_regressor(h, R, which, 3, B, matches_in, is_float, n, B.rowmap, B.d_count, matches_out, probs_out,
                       B.raw, st);
}

int p2p_refine_taps(p2p_handle_t h, int32_t* info_out, float* scales_out, int32_t* rows_out, void* y_hi, void* y_lo,
                    float* pooled, void* h1_hi, void* h1_lo, void* h2_hi, void* h2_lo, float* raw_out, void* stream) {
  P2P_ENTER(h);
  P2P_REQUIRE(info_out && scales_out, "null info / scales pointer");
  const auto& T = h->tap;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  int m = T.n;
  if (T.d_count != nullptr) {
    P2P_CUDA_OK(cudaStreamSynchronize(st));
    P2P_CUDA_OK(cudaMemcpy(&m, T.d_count, sizeof(int), cudaMemcpyDeviceToHost));
  }
  info_out[0] = m;
  info_out[1] = T.passes;
  info_out[2] = T.d_count != nullptr;
  info_out[3] = T.fc_tc;
  for (int i = 0; i < 4; ++i) scales_out[i] = T.scales[i];
  if (T.n == 0) return 0;
  P2P_REQUIRE(!y_lo || T.passes == 3, "y_lo is written by 3-pass passes only");
  P2P_REQUIRE(!(h1_hi || h1_lo || h2_hi || h2_lo) || T.fc_tc, "h1 / h2 are written by the tensor-core FC only");
#define TAP(dst, src, bytes) \
  if (dst) P2P_CUDA_OK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, st))
  if (rows_out) {
    if (T.rowmap != nullptr) {
      TAP(rows_out, T.rowmap, (size_t)m * 4);
    } else {
      std::vector<int32_t> id(m);
      for (int i = 0; i < m; ++i) id[i] = i;
      P2P_CUDA_OK(cudaMemcpy(rows_out, id.data(), (size_t)m * 4, cudaMemcpyHostToDevice));
    }
  }
  TAP(y_hi, T.y_hi, (size_t)m * 64 * 512 * 2);
  TAP(y_lo, T.y_lo, (size_t)m * 64 * 512 * 2);
  TAP(pooled, T.pooled, (size_t)m * 512 * 4);
  TAP(h1_hi, T.h1_hi, (size_t)m * 512 * 2);
  TAP(h1_lo, T.h1_lo, (size_t)m * 512 * 2);
  TAP(h2_hi, T.h2_hi, (size_t)m * 256 * 2);
  TAP(h2_lo, T.h2_lo, (size_t)m * 256 * 2);
  TAP(raw_out, T.raw, (size_t)T.n * 5 * 4);
#undef TAP
  return 0;
}

int p2p_finalize_matches(p2p_handle_t h, const float* fine, const float* scores, const int64_t* coarse, int n, float io_thres,
                         const double* upscale4, double* packed_out, void* stream) {
  P2P_ENTER(h);
  P2P_REQUIRE(scores && coarse && upscale4 && packed_out && n >= 0, "bad argument");
  return launch_finalize_matches(fine, scores, (const long long*)coarse, n, io_thres, upscale4, packed_out,
                                 reinterpret_cast<cudaStream_t>(stream));
}

static int preprocess_impl(p2p_handle_t h, const uint8_t* rgb_hwc, int ho, int wo, int ht, int wt, float* out_chw,
                           uint8_t* resized_hwc_out, float* gray_hw, void* stream) {
  P2P_ENTER(h);
  P2P_REQUIRE(rgb_hwc && out_chw && ho > 0 && wo > 0 && ht > 0 && wt > 0, "bad argument");
  P2P_REQUIRE((long long)ho * wo < (1ll << 28) && (long long)ht * wt < (1ll << 28), "image too large");
  const PreprocessCoefs* C = nullptr;
  for (const auto& c : h->pre_coefs)
    if (c.ho == ho && c.wo == wo && c.ht == ht && c.wt == wt) C = &c;
  if (C == nullptr) {
    if (h->pre_coefs.size() >= 32) {            // drop the oldest table (nothing may still be reading it)
      P2P_CUDA_OK(cudaDeviceSynchronize());
      if (h->pre_coefs.front().d) cudaFree(h->pre_coefs.front().d);
      h->pre_coefs.erase(h->pre_coefs.begin());
    }
    PreprocessCoefs c;
    int rc = preprocess_build_coefs(ho, wo, ht, wt, c);
    if (rc) return rc;
    h->pre_coefs.push_back(c);
    C = &h->pre_coefs.back();
  }
  int rc = h->pre.reserve((size_t)ho * wt * 3 + 4096);
  if (rc) return rc;
  uint8_t* tmp = (uint8_t*)h->pre.take((size_t)ho * wt * 3);
  P2P_REQUIRE(tmp != nullptr, "scratch carve failed");
  const float mean[3] = {0.485f, 0.456f, 0.406f}, stdv[3] = {0.229f, 0.224f, 0.225f};   // ImageNet, preprocess.py:93
  return launch_preprocess(rgb_hwc, *C, mean, stdv, out_chw, resized_hwc_out, gray_hw, tmp,
                           reinterpret_cast<cudaStream_t>(stream));
}

int p2p_preprocess_image(p2p_handle_t h, const uint8_t* rgb_hwc, int ho, int wo, int ht, int wt, float* out_chw,
                         uint8_t* resized_hwc_out, void* stream) {
  return preprocess_impl(h, rgb_hwc, ho, wo, ht, wt, out_chw, resized_hwc_out, nullptr, stream);
}

int p2p_preprocess_image_gray(p2p_handle_t h, const uint8_t* rgb_hwc, int ho, int wo, int ht, int wt, float* out_chw,
                              float* gray_hw, void* stream) {
  return preprocess_impl(h, rgb_hwc, ho, wo, ht, wt, out_chw, nullptr, gray_hw, stream);
}

int p2p_find_model(p2p_handle_t h, int model, const double* rows, int row_stride, int n, const double* n_dev, double px_th,
                   double conf, int max_iters, unsigned long long seed, double* model_out, uint8_t* mask_out,
                   int32_t* n_inliers_out, void* stream) {
  P2P_ENTER(h);
  P2P_REQUIRE(model >= 0 && model <= 2, "model must be 0 (F), 1 (H) or 2 (F with the DEGENSAC degeneracy check)");
  P2P_REQUIRE(model_out && mask_out && n_inliers_out && (rows || n == 0), "null tensor pointer");
  P2P_REQUIRE(n >= 0 && n <= (1 << 26) && row_stride >= 4, "bad row count or stride");
  P2P_REQUIRE(px_th > 0.0 && isfinite(px_th), "px_th must be positive");
  P2P_REQUIRE(conf > 0.0 && conf < 1.0, "conf must lie in (0, 1)");
  P2P_REQUIRE(max_iters > 0 && max_iters <= (1 << 24), "max_iters must lie in [1, 2^24]");
  int rc = h->verify.reserve(verify_scratch_bytes(1, n, true) + 4096);
  if (rc) return rc;
  void* scratch = h->verify.take(verify_scratch_bytes(1, n, true));
  return launch_find_model(model, single_pair(rows, row_stride, n, n_dev), px_th, conf, max_iters, seed, scratch,
                           model_out, mask_out, n_inliers_out, reinterpret_cast<cudaStream_t>(stream));
}

// ---- batches of pairs: validation of the host copy of the offsets and the split into launches ------------------------
static int check_batch(const double* rows, int row_stride, const int64_t* offsets, const int64_t* offsets_host, int K) {
  P2P_REQUIRE(K >= 0, "K must be non-negative");
  P2P_REQUIRE(row_stride >= 4, "row_stride must be at least 4");
  if (K == 0) return 0;
  P2P_REQUIRE(offsets && offsets_host, "null offsets pointer");
  P2P_REQUIRE(offsets_host[0] >= 0, "offsets must be non-negative");
  for (int k = 0; k < K; ++k) {
    const int64_t len = offsets_host[k + 1] - offsets_host[k];
    P2P_REQUIRE(len >= 0, "offsets must be non-decreasing");
    P2P_REQUIRE(len <= (1 << 26), "a pair has more than 2^26 rows");
  }
  P2P_REQUIRE(offsets_host[K] - offsets_host[0] < ((int64_t)1 << 31), "a batch must have fewer than 2^31 rows");
  P2P_REQUIRE(rows || offsets_host[K] == offsets_host[0], "null rows pointer");
  return 0;
}

// Pairs k0 .. k0 + pairs - 1 of a batch as one launch.
static PairBatch batch_chunk(const double* rows, int row_stride, const int64_t* offsets, const int64_t* offsets_host,
                             const double* n_dev, int k0, int pairs) {
  return PairBatch{rows, row_stride, reinterpret_cast<const long long*>(offsets) + k0, 0,
                   n_dev ? n_dev + k0 : nullptr, (long long)offsets_host[k0],
                   (long long)(offsets_host[k0 + pairs] - offsets_host[k0]), pairs};
}

// Largest scratch of any launch of `chunk` pairs.
static size_t batch_scratch(const int64_t* offsets_host, int K, int chunk, size_t (*bytes)(int, long long)) {
  size_t need = 0;
  for (int k0 = 0; k0 < K; k0 += chunk) {
    const int pairs = std::min(chunk, K - k0);
    need = std::max(need, bytes(pairs, (long long)(offsets_host[k0 + pairs] - offsets_host[k0])));
  }
  return need;
}

int p2p_batch_chunk_pairs(p2p_handle_t h, int entry, int* pairs_out) {
  P2P_ENTER(h);
  P2P_REQUIRE(pairs_out != nullptr, "null pointer");
  P2P_REQUIRE(entry >= 0 && entry <= 3,
              "entry must be 0 (find_model), 1 (find_essential), 2 (recover_pose) or 3 (find_absolute_pose)");
  *pairs_out = entry == 0   ? verify_chunk_pairs()
               : entry == 1 ? essential_chunk_pairs()
               : entry == 2 ? pose_chunk_pairs()
                            : abspose_chunk_queries();
  return 0;
}

int p2p_find_model_batch(p2p_handle_t h, int model, const double* rows, int row_stride, const int64_t* offsets,
                         const int64_t* offsets_host, int K, const double* n_dev, double px_th, double conf, int max_iters,
                         unsigned long long seed, double* models_out, uint8_t* mask_out, int32_t* n_inliers_out,
                         void* stream) {
  P2P_ENTER(h);
  P2P_REQUIRE(model >= 0 && model <= 2, "model must be 0 (F), 1 (H) or 2 (F with the DEGENSAC degeneracy check)");
  int rc = check_batch(rows, row_stride, offsets, offsets_host, K);
  if (rc) return rc;
  P2P_REQUIRE(px_th > 0.0 && isfinite(px_th), "px_th must be positive");
  P2P_REQUIRE(conf > 0.0 && conf < 1.0, "conf must lie in (0, 1)");
  P2P_REQUIRE(max_iters > 0 && max_iters <= (1 << 24), "max_iters must lie in [1, 2^24]");
  if (K == 0) return 0;
  P2P_REQUIRE(models_out && mask_out && n_inliers_out, "null tensor pointer");
  const int chunk = verify_chunk_pairs();
  const size_t need = batch_scratch(offsets_host, K, chunk, [](int p, long long r) { return verify_scratch_bytes(p, r, true); });
  if ((rc = h->verify.reserve(need + 4096))) return rc;
  void* scratch = h->verify.take(need);
  for (int k0 = 0; k0 < K; k0 += chunk) {
    const PairBatch B = batch_chunk(rows, row_stride, offsets, offsets_host, n_dev, k0, std::min(chunk, K - k0));
    if ((rc = launch_find_model(model, B, px_th, conf, max_iters, seed, scratch, models_out + 9 * (size_t)k0, mask_out,
                                n_inliers_out + k0, reinterpret_cast<cudaStream_t>(stream))))
      return rc;
  }
  return 0;
}

int p2p_sampson_distance(p2p_handle_t h, const double* rows, int row_stride, int n, const double* F, double* dist_out,
                         void* stream) {
  P2P_ENTER(h);
  P2P_REQUIRE(F && dist_out && (rows || n == 0), "null tensor pointer");
  P2P_REQUIRE(n >= 0 && row_stride >= 4, "bad row count or stride");
  return launch_sampson_distance(rows, row_stride, n, F, dist_out, reinterpret_cast<cudaStream_t>(stream));
}

int p2p_epipolar_histograms(p2p_handle_t h, const double* rows, int row_stride, int n, const double* n_dev,
                            int coarse_col, const double* F, const uint8_t* mask, const double* edges, int n_edges,
                            int32_t* counts_out, void* stream) {
  P2P_ENTER(h);
  P2P_REQUIRE(F && edges && counts_out && (rows || n == 0), "null pointer");
  P2P_REQUIRE(n >= 0 && row_stride >= 4, "bad row count or stride");
  P2P_REQUIRE(coarse_col == -1 || (coarse_col >= 0 && coarse_col + 4 <= row_stride),
              "coarse_col must be -1 or a column with 4 columns of the row from it");
  P2P_REQUIRE(n_edges >= 2 && n_edges <= kMaxHistEdges, "n_edges must be in 2..16");
  EpiHistArgs a{};
  for (int j = 0; j < 9; ++j) a.F[j] = F[j];
  for (int i = 0; i < n_edges; ++i) {
    P2P_REQUIRE(std::isfinite(edges[i]) && (i == 0 || edges[i] > edges[i - 1]), "edges must be finite and increasing");
    a.edges[i] = edges[i];
  }
  a.n_edges = n_edges;
  return launch_epipolar_histograms(rows, row_stride, n, n_dev, coarse_col, mask, a, counts_out,
                                    reinterpret_cast<cudaStream_t>(stream));
}

int p2p_homography_errors(p2p_handle_t h, const double* rows, int row_stride, int n, const double* n_dev,
                          const double* H_gt, const double* H_pred, int width, int height, const double* thresholds,
                          int n_thr, int32_t* counts_out, double* corner_err_out, void* stream) {
  P2P_ENTER(h);
  P2P_REQUIRE(H_gt && H_pred && thresholds && counts_out && corner_err_out && (rows || n == 0), "null pointer");
  P2P_REQUIRE(n >= 0 && row_stride >= 4, "bad row count or stride");
  P2P_REQUIRE(width >= 1 && height >= 1, "width and height must be positive");
  P2P_REQUIRE(n_thr >= 1 && n_thr <= kMaxHomThresholds, "n_thr must be in 1..16");
  HomErrArgs a{};
  for (int j = 0; j < 9; ++j) a.H[j] = H_gt[j];
  for (int i = 0; i < kMaxHomThresholds; ++i) a.thr[i] = NAN;     // no row passes a padding entry
  for (int i = 0; i < n_thr; ++i) {
    P2P_REQUIRE(std::isfinite(thresholds[i]) && thresholds[i] > 0.0 && (i == 0 || thresholds[i] > thresholds[i - 1]),
                "thresholds must be finite, positive and strictly increasing");
    a.thr[i] = thresholds[i];
  }
  a.n_thr = n_thr;
  a.width = width;
  a.height = height;
  return launch_homography_errors(rows, row_stride, n, n_dev, a, H_pred, counts_out, corner_err_out,
                                  reinterpret_cast<cudaStream_t>(stream));
}

int p2p_overlap_scores(p2p_handle_t h, const int64_t* point3D_ids, const int64_t* offsets,
                       const int64_t* offsets_host, int n_images, int words, uint32_t* bits_out, int32_t* counts_out,
                       double* scores_out, void* stream) {
  P2P_ENTER(h);
  P2P_REQUIRE(n_images >= 0 && n_images <= kMaxOverlapImages, "n_images must be in 0 .. 2^20");
  P2P_REQUIRE(words >= 0 && words <= (int)((kMaxOverlapPoints + 31) / 32), "words must be in 0 .. 2^26");
  P2P_REQUIRE(offsets_host != nullptr, "offsets_host is null");
  if (n_images == 0) return 0;
  P2P_REQUIRE(offsets && counts_out && scores_out && (bits_out || words == 0), "null pointer");
  P2P_REQUIRE(offsets_host[0] >= 0, "offsets must be non-negative");
  for (int i = 0; i < n_images; ++i) {
    const int64_t len = offsets_host[i + 1] - offsets_host[i];
    P2P_REQUIRE(len >= 0, "offsets must be non-decreasing");
    P2P_REQUIRE(len <= kMaxOverlapPoints, "an image has 2^31 or more 2D points");
    P2P_REQUIRE((len + 31) / 32 <= words, "words is smaller than ceil(n2d / 32) of an image");
  }
  P2P_REQUIRE(point3D_ids || offsets_host[n_images] == offsets_host[0], "point3D_ids is null");
  return launch_overlap_scores(reinterpret_cast<const long long*>(point3D_ids),
                               reinterpret_cast<const long long*>(offsets), n_images, words,
                               reinterpret_cast<unsigned*>(bits_out), counts_out, scores_out,
                               reinterpret_cast<cudaStream_t>(stream));
}

int p2p_test_hypotheses(p2p_handle_t h, int model, const double* rows, int row_stride, int n, double px_th,
                        unsigned long long seed, int count, double* models_out, int32_t* counts_out, void* stream) {
  P2P_ENTER(h);
  P2P_REQUIRE(model == 0 || model == 1, "model must be 0 (F) or 1 (H)");
  P2P_REQUIRE(rows && models_out && counts_out && count > 0 && row_stride >= 4, "bad argument");
  P2P_REQUIRE(n >= (model == 0 ? 7 : 4) && n <= (1 << 26), "fewer rows than a minimal sample");
  int rc = h->verify.reserve(verify_scratch_bytes(1, n, false) + 4096);
  if (rc) return rc;
  void* scratch = h->verify.take(verify_scratch_bytes(1, n, false));
  return launch_test_hypotheses(model, rows, row_stride, n, px_th, seed, count, scratch, models_out, counts_out,
                                reinterpret_cast<cudaStream_t>(stream));
}

int p2p_test_degeneracy(p2p_handle_t h, const double* rows, int row_stride, int n, double px_th, unsigned long long seed,
                        int count, int32_t* triplet_out, double* H_out, void* stream) {
  P2P_ENTER(h);
  P2P_REQUIRE(rows && triplet_out && H_out && count > 0 && count <= (1 << 20) && row_stride >= 4, "bad argument");
  P2P_REQUIRE(n >= 7 && n <= (1 << 26), "fewer rows than a minimal sample");
  P2P_REQUIRE(px_th > 0.0 && isfinite(px_th), "px_th must be positive");
  int rc = h->verify.reserve(verify_degeneracy_scratch_bytes(n, count) + 4096);
  if (rc) return rc;
  void* scratch = h->verify.take(verify_degeneracy_scratch_bytes(n, count));
  return launch_test_degeneracy(rows, row_stride, n, px_th, seed, count, scratch, triplet_out, H_out,
                                reinterpret_cast<cudaStream_t>(stream));
}

static bool intrinsics_ok(const double* intr, Intrinsics& K) {
  if (intr == nullptr) return false;
  for (int i = 0; i < 8; ++i)
    if (!isfinite(intr[i])) return false;
  K = Intrinsics{intr[0], intr[1], intr[2], intr[3], intr[4], intr[5], intr[6], intr[7]};
  return K.fx1 > 0.0 && K.fy1 > 0.0 && K.fx2 > 0.0 && K.fy2 > 0.0;
}

int p2p_find_essential(p2p_handle_t h, const double* rows, int row_stride, int n, const double* n_dev, const double* intr,
                       double px_th, double conf, int max_iters, unsigned long long seed, double* E_out, uint8_t* mask_out,
                       int32_t* n_inliers_out, void* stream) {
  P2P_ENTER(h);
  P2P_REQUIRE(E_out && mask_out && n_inliers_out && (rows || n == 0), "null tensor pointer");
  P2P_REQUIRE(n >= 0 && n <= (1 << 26) && row_stride >= 4, "bad row count or stride");
  Intrinsics K;
  P2P_REQUIRE(intrinsics_ok(intr, K), "intr must be 8 finite values with positive focal lengths");
  P2P_REQUIRE(px_th > 0.0 && isfinite(px_th), "px_th must be positive");
  P2P_REQUIRE(conf > 0.0 && conf < 1.0, "conf must lie in (0, 1)");
  P2P_REQUIRE(max_iters > 0 && max_iters <= (1 << 24), "max_iters must lie in [1, 2^24]");
  int rc = h->verify.reserve(essential_scratch_bytes(1, n, true) + 4096);
  if (rc) return rc;
  void* scratch = h->verify.take(essential_scratch_bytes(1, n, true));
  return launch_find_essential(single_pair(rows, row_stride, n, n_dev), nullptr, K, px_th, nullptr, conf, max_iters,
                               seed, scratch, E_out, mask_out, n_inliers_out, reinterpret_cast<cudaStream_t>(stream));
}

// p2p_find_essential_batch with one px_th for every pair (px_th_dev null), or with pair k's at px_th_dev[k].
static int find_essential_batch(p2p_handle_t h, const double* rows, int row_stride, const int64_t* offsets,
                                const int64_t* offsets_host, int K, const double* n_dev, const double* intr,
                                double px_th, const double* px_th_dev, double conf, int max_iters,
                                unsigned long long seed, double* E_out, uint8_t* mask_out, int32_t* n_inliers_out,
                                void* stream) {
  int rc = check_batch(rows, row_stride, offsets, offsets_host, K);
  if (rc) return rc;
  P2P_REQUIRE(px_th_dev != nullptr || (px_th > 0.0 && isfinite(px_th)), "px_th must be positive");
  P2P_REQUIRE(conf > 0.0 && conf < 1.0, "conf must lie in (0, 1)");
  P2P_REQUIRE(max_iters > 0 && max_iters <= (1 << 24), "max_iters must lie in [1, 2^24]");
  if (K == 0) return 0;
  P2P_REQUIRE(intr && E_out && mask_out && n_inliers_out, "null tensor pointer");
  const int chunk = essential_chunk_pairs();
  const size_t need =
      batch_scratch(offsets_host, K, chunk, [](int p, long long r) { return essential_scratch_bytes(p, r, true); });
  if ((rc = h->verify.reserve(need + 4096))) return rc;
  void* scratch = h->verify.take(need);
  for (int k0 = 0; k0 < K; k0 += chunk) {
    const PairBatch B = batch_chunk(rows, row_stride, offsets, offsets_host, n_dev, k0, std::min(chunk, K - k0));
    if ((rc = launch_find_essential(B, intr + 8 * (size_t)k0, Intrinsics{}, px_th,
                                    px_th_dev ? px_th_dev + k0 : nullptr, conf, max_iters, seed, scratch,
                                    E_out + 9 * (size_t)k0, mask_out, n_inliers_out + k0,
                                    reinterpret_cast<cudaStream_t>(stream))))
      return rc;
  }
  return 0;
}

int p2p_find_essential_batch(p2p_handle_t h, const double* rows, int row_stride, const int64_t* offsets,
                             const int64_t* offsets_host, int K, const double* n_dev, const double* intr, double px_th,
                             double conf, int max_iters, unsigned long long seed, double* E_out, uint8_t* mask_out,
                             int32_t* n_inliers_out, void* stream) {
  P2P_ENTER(h);
  return find_essential_batch(h, rows, row_stride, offsets, offsets_host, K, n_dev, intr, px_th, nullptr, conf,
                              max_iters, seed, E_out, mask_out, n_inliers_out, stream);
}

int p2p_find_essential_batch_th(p2p_handle_t h, const double* rows, int row_stride, const int64_t* offsets,
                                const int64_t* offsets_host, int K, const double* n_dev, const double* intr,
                                const double* px_th, double conf, int max_iters, unsigned long long seed,
                                double* E_out, uint8_t* mask_out, int32_t* n_inliers_out, void* stream) {
  P2P_ENTER(h);
  P2P_REQUIRE(px_th != nullptr, "null px_th pointer");
  return find_essential_batch(h, rows, row_stride, offsets, offsets_host, K, n_dev, intr, 0.0, px_th, conf, max_iters,
                              seed, E_out, mask_out, n_inliers_out, stream);
}

int p2p_recover_pose(p2p_handle_t h, const double* rows, int row_stride, int n, const double* n_dev, const double* intr,
                     const double* E, const uint8_t* mask_in, double dist_th, double* Rt_out, uint8_t* mask_out,
                     int32_t* n_good_out, void* stream) {
  P2P_ENTER(h);
  P2P_REQUIRE(E && Rt_out && mask_out && n_good_out && (rows || n == 0), "null tensor pointer");
  P2P_REQUIRE(n >= 0 && n <= (1 << 26) && row_stride >= 4, "bad row count or stride");
  Intrinsics K;
  P2P_REQUIRE(intrinsics_ok(intr, K), "intr must be 8 finite values with positive focal lengths");
  P2P_REQUIRE(dist_th > 0.0 && isfinite(dist_th), "dist_th must be positive");
  int rc = h->verify.reserve(pose_scratch_bytes(1, n) + 4096);
  if (rc) return rc;
  void* scratch = h->verify.take(pose_scratch_bytes(1, n));
  return launch_recover_pose(single_pair(rows, row_stride, n, n_dev), nullptr, K, E, mask_in, dist_th, scratch, Rt_out,
                             mask_out, n_good_out, reinterpret_cast<cudaStream_t>(stream));
}

int p2p_recover_pose_batch(p2p_handle_t h, const double* rows, int row_stride, const int64_t* offsets,
                           const int64_t* offsets_host, int K, const double* n_dev, const double* intr, const double* E,
                           const uint8_t* mask_in, double dist_th, double* Rt_out, uint8_t* mask_out, int32_t* n_good_out,
                           void* stream) {
  P2P_ENTER(h);
  int rc = check_batch(rows, row_stride, offsets, offsets_host, K);
  if (rc) return rc;
  P2P_REQUIRE(dist_th > 0.0 && isfinite(dist_th), "dist_th must be positive");
  if (K == 0) return 0;
  P2P_REQUIRE(intr && E && Rt_out && mask_out && n_good_out, "null tensor pointer");
  const int chunk = pose_chunk_pairs();
  const size_t need = batch_scratch(offsets_host, K, chunk, [](int p, long long r) { return pose_scratch_bytes(p, r); });
  if ((rc = h->verify.reserve(need + 4096))) return rc;
  void* scratch = h->verify.take(need);
  for (int k0 = 0; k0 < K; k0 += chunk) {
    const PairBatch B = batch_chunk(rows, row_stride, offsets, offsets_host, n_dev, k0, std::min(chunk, K - k0));
    if ((rc = launch_recover_pose(B, intr + 8 * (size_t)k0, Intrinsics{}, E + 9 * (size_t)k0, mask_in, dist_th, scratch,
                                  Rt_out + 12 * (size_t)k0, mask_out, n_good_out + k0,
                                  reinterpret_cast<cudaStream_t>(stream))))
      return rc;
  }
  return 0;
}

int p2p_relpose_errors_batch(p2p_handle_t h, const double* rows, int row_stride, const int64_t* offsets,
                             const int64_t* offsets_host, int K, const double* n_dev, const double* intr,
                             const double* Rt_gt, const double* Rt_est, const int32_t* n_inliers,
                             const double* thresholds, int n_thr, double* out, int out_stride, void* stream) {
  P2P_ENTER(h);
  int rc = check_batch(rows, row_stride, offsets, offsets_host, K);
  if (rc) return rc;
  P2P_REQUIRE(thresholds != nullptr, "null thresholds pointer");
  P2P_REQUIRE(n_thr >= 1 && n_thr <= kMaxRelposeThresholds, "n_thr must be in 1..16");
  P2P_REQUIRE(out_stride >= 2 + (n_thr + 2) / 2, "out_stride must hold 2 doubles and n_thr + 1 int32 counts");
  RelposeErrArgs a{};
  for (int i = 0; i < kMaxRelposeThresholds; ++i) a.thr[i] = NAN;     // no row passes a padding entry
  for (int i = 0; i < n_thr; ++i) {
    P2P_REQUIRE(std::isfinite(thresholds[i]) && thresholds[i] > 0.0 && (i == 0 || thresholds[i] > thresholds[i - 1]),
                "thresholds must be finite, positive and strictly increasing");
    a.thr[i] = thresholds[i];
  }
  a.n_thr = n_thr;
  if (K == 0) return 0;
  P2P_REQUIRE(intr && Rt_gt && Rt_est && n_inliers && out, "null tensor pointer");
  return launch_relpose_errors(batch_chunk(rows, row_stride, offsets, offsets_host, n_dev, 0, K), intr, Rt_gt, Rt_est,
                               n_inliers, a, out, out_stride, reinterpret_cast<cudaStream_t>(stream));
}

int p2p_test_essential_hypotheses(p2p_handle_t h, const double* rows, int row_stride, int n, const double* intr,
                                  double px_th, unsigned long long seed, int count, double* models_out,
                                  int32_t* counts_out, void* stream) {
  P2P_ENTER(h);
  P2P_REQUIRE(rows && models_out && counts_out && count > 0 && row_stride >= 4, "bad argument");
  P2P_REQUIRE(n >= 5 && n <= (1 << 26), "fewer rows than a minimal sample");
  Intrinsics K;
  P2P_REQUIRE(intrinsics_ok(intr, K), "intr must be 8 finite values with positive focal lengths");
  P2P_REQUIRE(px_th > 0.0 && isfinite(px_th), "px_th must be positive");
  int rc = h->verify.reserve(essential_scratch_bytes(1, n, false) + 4096);
  if (rc) return rc;
  void* scratch = h->verify.take(essential_scratch_bytes(1, n, false));
  return launch_test_essential_hypotheses(rows, row_stride, n, K, px_th, seed, count, scratch, models_out, counts_out,
                                          reinterpret_cast<cudaStream_t>(stream));
}

int p2p_find_absolute_pose_batch(p2p_handle_t h, const double* rows, int row_stride, const int64_t* offsets,
                                 const int64_t* offsets_host, int K, const double* n_dev, const double* intr,
                                 double px_th, const double* px_th_dev, double conf, int max_iters,
                                 unsigned long long seed, double* Rt_out, uint8_t* mask_out, int32_t* n_inliers_out,
                                 void* stream) {
  P2P_ENTER(h);
  P2P_REQUIRE(row_stride >= 5, "row_stride must be at least 5");
  int rc = check_batch(rows, row_stride, offsets, offsets_host, K);
  if (rc) return rc;
  P2P_REQUIRE(px_th_dev != nullptr || (px_th > 0.0 && isfinite(px_th)), "px_th must be positive");
  P2P_REQUIRE(conf > 0.0 && conf < 1.0, "conf must lie in (0, 1)");
  P2P_REQUIRE(max_iters > 0 && max_iters <= (1 << 24), "max_iters must lie in [1, 2^24]");
  if (K == 0) return 0;
  P2P_REQUIRE(intr && Rt_out && mask_out && n_inliers_out, "null tensor pointer");
  const int chunk = abspose_chunk_queries();
  const size_t need =
      batch_scratch(offsets_host, K, chunk, [](int p, long long r) { return abspose_scratch_bytes(p, r, true); });
  if ((rc = h->verify.reserve(need + 4096))) return rc;
  void* scratch = h->verify.take(need);
  for (int k0 = 0; k0 < K; k0 += chunk) {
    const PairBatch B = batch_chunk(rows, row_stride, offsets, offsets_host, n_dev, k0, std::min(chunk, K - k0));
    if ((rc = launch_find_absolute_pose(B, intr + 4 * (size_t)k0, px_th, px_th_dev ? px_th_dev + k0 : nullptr, conf,
                                        max_iters, seed, scratch, Rt_out + 12 * (size_t)k0, mask_out,
                                        n_inliers_out + k0, reinterpret_cast<cudaStream_t>(stream))))
      return rc;
  }
  return 0;
}

int p2p_test_absolute_pose_hypotheses(p2p_handle_t h, const double* rows, int row_stride, int n, const double* intr,
                                      double px_th, unsigned long long seed, int count, double* models_out,
                                      int32_t* counts_out, void* stream) {
  P2P_ENTER(h);
  P2P_REQUIRE(rows && models_out && counts_out && count > 0 && count <= (1 << 20) && row_stride >= 5, "bad argument");
  P2P_REQUIRE(n >= 4 && n <= (1 << 26), "fewer than 4 rows");
  P2P_REQUIRE(intr != nullptr && isfinite(intr[0]) && isfinite(intr[1]) && isfinite(intr[2]) && isfinite(intr[3]) &&
                  intr[0] > 0.0 && intr[1] > 0.0,
              "intr must be 4 finite values with positive focal lengths");
  P2P_REQUIRE(px_th > 0.0 && isfinite(px_th), "px_th must be positive");
  int rc = h->verify.reserve(abspose_scratch_bytes(1, n, false) + 4096);
  if (rc) return rc;
  void* scratch = h->verify.take(abspose_scratch_bytes(1, n, false));
  return launch_test_absolute_pose_hypotheses(rows, row_stride, n, intr, px_th, seed, count, scratch, models_out,
                                              counts_out, reinterpret_cast<cudaStream_t>(stream));
}

int p2p_lift_scan(p2p_handle_t h, const double* scan, int height, int width, const double* align,
                  const double* matches, int match_stride, int n, const double* n_dev, double* rows_out,
                  int row_stride, long long capacity, double* count_dev, void* stream) {
  P2P_ENTER(h);
  P2P_REQUIRE(height >= 1 && width >= 1 && (size_t)height * width <= ((size_t)1 << 31), "bad scan size");
  P2P_REQUIRE(match_stride >= 4 && row_stride >= 5, "match_stride must be at least 4 and row_stride at least 5");
  P2P_REQUIRE(n >= 0 && n <= (1 << 26) && capacity >= 0, "bad match count or capacity");
  P2P_REQUIRE(align != nullptr, "null alignment");
  for (int i = 0; i < 16; ++i) P2P_REQUIRE(std::isfinite(align[i]), "the alignment must be finite");
  P2P_REQUIRE(scan && count_dev && (matches || n == 0) && (rows_out || capacity == 0), "null pointer");
  if (n == 0) return 0;
  return launch_lift_scan(scan, height, width, align, matches, match_stride, n, n_dev, rows_out, row_stride, capacity,
                          count_dev, reinterpret_cast<cudaStream_t>(stream));
}

int p2p_sfm_keypoints(p2p_handle_t h, const double* matches, long long n_matches, const int64_t* offsets, int n_pairs,
                      const int32_t* pair_img, int both_sides, double merge_px, double* kp_xy, uint64_t* kp_key,
                      int32_t* kp_of_ep, int64_t* counts, void* stream) {
  P2P_ENTER(h);
  P2P_REQUIRE(n_matches >= 0 && n_matches <= (1ll << 30) && n_pairs >= 1 && n_pairs < (1 << 30), "bad match count");
  P2P_REQUIRE(both_sides == 0 || both_sides == 1, "both_sides must be 0 or 1");
  P2P_REQUIRE(merge_px > 0.0 && std::isfinite(merge_px), "merge_px must be positive");
  P2P_REQUIRE(offsets && pair_img && counts && kp_xy && kp_key && kp_of_ep && (matches || n_matches == 0),
              "null pointer");
  return launch_sfm_keypoints(h->sfm, matches, n_matches, (const long long*)offsets, n_pairs, pair_img, both_sides,
                              merge_px, kp_xy, (unsigned long long*)kp_key, kp_of_ep, (long long*)counts,
                              reinterpret_cast<cudaStream_t>(stream));
}

int p2p_sfm_undistort(p2p_handle_t h, const double* xy, const uint64_t* kp_key, long long capacity,
                      const int64_t* n_dev, const int32_t* img_cam, const double* cams, double* xy_out, void* stream) {
  P2P_ENTER(h);
  P2P_REQUIRE(capacity >= 0 && capacity <= (1ll << 31), "bad capacity");
  P2P_REQUIRE((xy && kp_key && img_cam && cams && xy_out) || capacity == 0, "null pointer");
  return launch_sfm_undistort(xy, (const unsigned long long*)kp_key, capacity, (const long long*)n_dev, img_cam, cams,
                              xy_out, reinterpret_cast<cudaStream_t>(stream));
}

int p2p_sfm_tracks(p2p_handle_t h, const int32_t* kp_of_ep, long long n_matches, const int64_t* offsets, int n_pairs,
                   const double* E, const double* thr, const double* kp_n, long long n_kp, int32_t* labels,
                   int32_t* obs_kp, int32_t* track_start, int32_t* track_len, int64_t* counts_dev, int64_t* counts_host,
                   void* stream) {
  P2P_ENTER(h);
  P2P_REQUIRE(n_matches >= 0 && n_matches <= (1ll << 30) && n_pairs >= 1 && n_kp >= 0 && n_kp < (1ll << 31) - 1,
              "bad sizes");
  P2P_REQUIRE(offsets && counts_dev && counts_host && (n_matches == 0 || (kp_of_ep && E && thr && kp_n)) &&
                  (n_kp == 0 || (labels && obs_kp && track_start && track_len)),
              "null pointer");
  return launch_sfm_tracks(h->sfm, kp_of_ep, n_matches, (const long long*)offsets, n_pairs, E, thr, kp_n, n_kp, labels,
                           obs_kp, track_start, track_len, (long long*)counts_dev, (long long*)counts_host,
                           reinterpret_cast<cudaStream_t>(stream));
}

int p2p_sfm_triangulate(p2p_handle_t h, const int32_t* obs_kp, const int32_t* track_start, const int32_t* track_len,
                        int n_tracks, long long n_kp, const double* kp_xy, const double* kp_n, const uint64_t* kp_key,
                        const double* images, const int32_t* img_cam, const double* cams, double reproj_px,
                        double cos_min_angle, double* points, int32_t* point_len, double* point_err, int32_t* kp_point,
                        int64_t* counts, void* stream) {
  P2P_ENTER(h);
  P2P_REQUIRE(n_tracks >= 0 && n_tracks <= (1 << 27) && n_kp >= 0 && n_kp < (1ll << 31) - 1, "bad sizes");
  P2P_REQUIRE(reproj_px > 0.0 && std::isfinite(reproj_px), "reproj_px must be positive");
  P2P_REQUIRE(cos_min_angle > -1.0 && cos_min_angle <= 1.0, "cos_min_angle must lie in (-1, 1]");
  P2P_REQUIRE(counts && (n_kp == 0 || kp_point) &&
                  (n_tracks == 0 || (obs_kp && track_start && track_len && kp_xy && kp_n && kp_key && images &&
                                     img_cam && cams && points && point_len && point_err)),
              "null pointer");
  return launch_sfm_triangulate(h->sfm, obs_kp, track_start, track_len, n_tracks, n_kp, kp_xy, kp_n,
                                (const unsigned long long*)kp_key, images, img_cam, cams, reproj_px,
                                cos_min_angle, points, point_len, point_err, kp_point,
                                (long long*)counts, reinterpret_cast<cudaStream_t>(stream));
}

int p2p_sfm_query_rows(p2p_handle_t h, const double* matches, long long n_matches, const int64_t* offsets, int n_pairs,
                       const int32_t* pair_img, int n_queries, double merge_px, const int32_t* qkp_of_ep,
                       const uint64_t* qkp_key, const double* qkp_n, const double* q_intr, const uint64_t* kp_key,
                       const double* kp_xy, const int32_t* kp_point, long long n_kp, const double* points, double* rows,
                       int64_t* q_offsets, void* stream) {
  P2P_ENTER(h);
  P2P_REQUIRE(n_matches >= 0 && n_matches <= (1ll << 30) && n_pairs >= 1 && n_queries >= 1 &&
                  n_queries < (1 << 20) && n_kp >= 0 && n_kp < (1ll << 31) - 1,
              "bad sizes");
  P2P_REQUIRE(merge_px > 0.0 && std::isfinite(merge_px), "merge_px must be positive");
  P2P_REQUIRE(q_offsets && (n_matches == 0 || (matches && offsets && pair_img && qkp_of_ep && qkp_key && qkp_n &&
                                               q_intr && rows && (n_kp == 0 || (kp_key && kp_xy && kp_point && points)))),
              "null pointer");
  return launch_sfm_query_rows(h->sfm, matches, n_matches, (const long long*)offsets, n_pairs, pair_img, n_queries,
                               merge_px, qkp_of_ep, (const unsigned long long*)qkp_key, qkp_n, q_intr,
                               (const unsigned long long*)kp_key, kp_xy, kp_point, n_kp, points, rows,
                               (long long*)q_offsets, reinterpret_cast<cudaStream_t>(stream));
}

int p2p_test_gemm(p2p_handle_t h, const float* a, const float* b, float* c, int M, int N, int K, int passes,
                  int seg_len, float in_scale, void* stream) {
  P2P_ENTER(h);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  P2P_REQUIRE(a && b && c && M > 0 && N > 0 && K > 0, "bad argument");
  P2P_REQUIRE(K % 64 == 0 && K / 64 <= kMaxKSteps, "K must be a multiple of 64 and at most 6144");
  P2P_REQUIRE(passes == 1 || passes == 3, "passes must be 1 or 3");
  const int mpad = (int)align_up(M, 128), npad = (int)align_up(N, 256);
  const size_t ab = (size_t)mpad * K * 2, bb = (size_t)npad * K * 2;
  int rc = h->misc.reserve(2 * (ab + bb) + (1 << 16));
  if (rc) return rc;
  __half* a_hi = (__half*)h->misc.take(ab);
  __half* a_lo = (__half*)h->misc.take(ab);
  __half* b_hi = (__half*)h->misc.take(bb);
  __half* b_lo = (__half*)h->misc.take(bb);
  P2P_CUDA_OK(cudaMemsetAsync(a_hi, 0, 2 * ab, st));
  P2P_CUDA_OK(cudaMemsetAsync(b_hi, 0, 2 * bb, st));
  if ((rc = launch_split_rows(a, a_hi, a_lo, (size_t)M * K, in_scale, st))) return rc;
  if ((rc = launch_split_rows(b, b_hi, b_lo, (size_t)N * K, in_scale, st))) return rc;
  UmmaGemmParams p;
  memset(&p, 0, sizeof(p));
  const uint64_t ad[5] = {(uint64_t)K, 1, 1, 1, (uint64_t)mpad};
  const uint64_t as[4] = {(uint64_t)K * 2, (uint64_t)K * 2, (uint64_t)K * 2, (uint64_t)K * 2};
  const uint32_t abx[5] = {64, 1, 1, 1, 128};
  const uint64_t bd[2] = {(uint64_t)K, (uint64_t)npad};
  const uint64_t bs[1] = {(uint64_t)K * 2};
  const uint32_t bbx[2] = {64, 128};
  if ((rc = make_tmap_fp16(&p.a_main_hi, a_hi, 5, ad, as, abx))) return rc;
  if ((rc = make_tmap_fp16(&p.a_main_lo, a_lo, 5, ad, as, abx))) return rc;
  if ((rc = make_tmap_fp16(&p.b_hi, b_hi, 2, bd, bs, bbx))) return rc;
  if ((rc = make_tmap_fp16(&p.b_lo, b_lo, 2, bd, bs, bbx))) return rc;
  p.a_rgb_hi = p.a_main_hi;
  p.a_rgb_lo = p.a_main_lo;
  p.nsteps = K / 64;
  for (int s = 0; s < p.nsteps; ++s) p.steps[s] = KStep{(short)(s * 64), 0, 0, 0, 0, 0, s * 64};
  p.m_tiles = mpad / 128;
  p.n_tiles = npad / 256;
  p.a_units_per_tile = 128;
  p.seg_len = seg_len;
  p.epi.c = c;
  p.epi.ldc = N;
  p.epi.m_rows = M;
  p.epi.n_cols = N;
  p.epi.alpha = 1.f / (in_scale * in_scale);
  if ((rc = set_trace(h, p, 24, st))) return rc;
  return launch_umma_gemm(p, EPI_PLAIN, passes, sms(h), st);
}

int p2p_tile_trace_read(p2p_handle_t h, int idx, int* tag, int* tiles, unsigned long long* out, int max_tiles) {
  P2P_ENTER(h);
  P2P_REQUIRE(tag != nullptr && tiles != nullptr, "null argument");
  P2P_REQUIRE(idx >= 0 && idx < (int)h->traces.size(), "tile trace index out of range");
  const auto& t = h->traces[idx];
  *tag = t.tag;
  *tiles = t.tiles;
  if (out != nullptr) {
    P2P_REQUIRE(max_tiles >= t.tiles, "tile trace: output too small");
    P2P_CUDA_OK(cudaDeviceSynchronize());
    P2P_CUDA_OK(cudaMemcpy(out, h->trace_buf + t.off, (size_t)t.tiles * kTraceStamps * sizeof(unsigned long long),
                           cudaMemcpyDeviceToHost));
  }
  return 0;
}


int p2p_sp_keypoints(p2p_handle_t h, const float* logits, int batch, int hc, int wc, int nms_radius, float threshold,
                     int border, int max_keypoints, float* score_map, float* keypoints, float* scores, int64_t* offsets,
                     void* stream) {
  P2P_ENTER(h);
  P2P_REQUIRE(batch >= 1 && hc >= 1 && wc >= 1 && (long long)batch * hc * wc * 64 < (1ll << 31),
              "batch * 8hc * 8wc must be in 1 .. 2^31 - 1");
  P2P_REQUIRE(batch <= 65535 && hc <= 65535 * 4, "batch must be <= 65535 and hc <= 262140 (launch grid limits)");
  P2P_REQUIRE(nms_radius >= 0 && nms_radius <= kSpMaxNmsRadius, "nms_radius must be in 0..16");
  P2P_REQUIRE(border >= 0, "border must be >= 0");
  P2P_REQUIRE(std::isfinite(threshold), "threshold must be finite");
  P2P_REQUIRE(logits && keypoints && scores && offsets, "null pointer");
  return launch_sp_keypoints(h->sp, logits, batch, hc, wc, nms_radius, threshold, border, max_keypoints, score_map,
                             keypoints, scores, (long long*)offsets, reinterpret_cast<cudaStream_t>(stream));
}

int p2p_sp_descriptors(p2p_handle_t h, const float* desc, int batch, int dim, int hc, int wc, const float* keypoints,
                       const int64_t* offsets, long long n, float* out, void* stream) {
  P2P_ENTER(h);
  P2P_REQUIRE(batch >= 1 && hc >= 1 && wc >= 1, "empty descriptor map");
  P2P_REQUIRE((long long)batch * hc * wc < (1ll << 31), "batch * hc * wc must be < 2^31");
  P2P_REQUIRE(dim >= 1 && dim <= kSpMaxDescDim, "dim must be in 1..512");
  P2P_REQUIRE(n >= 0 && n < (1ll << 31), "bad keypoint count");
  P2P_REQUIRE(desc && offsets && ((keypoints && out) || n == 0), "null pointer");
  return launch_sp_descriptors(h->sp, desc, batch, dim, hc, wc, keypoints, (const long long*)offsets, n, out,
                               reinterpret_cast<cudaStream_t>(stream));
}

int p2p_match_descriptors_batch(p2p_handle_t h, const float* d0, const float* d1, const int64_t* offsets0,
                                const int64_t* offsets1, const int64_t* offsets0_host, const int64_t* offsets1_host,
                                int n_pairs, int dim, int mutual, double min_sim, double ratio, int32_t* match,
                                double* sim, double* tc_sim, int32_t* tc_idx, double* eps, int32_t* n_fixed,
                                void* stream) {
  P2P_ENTER(h);
  P2P_REQUIRE(n_pairs >= 1 && n_pairs <= 65535, "n_pairs must be in 1..65535");
  P2P_REQUIRE(dim >= 16 && dim <= kMatchMaxDim && dim % 16 == 0, "dim must be a multiple of 16 in 16..1024");
  P2P_REQUIRE(mutual == 0 || mutual == 1, "mutual must be 0 or 1");
  P2P_REQUIRE(!std::isinf(min_sim), "min_sim must be finite (NaN: no test)");
  P2P_REQUIRE(std::isnan(ratio) || (ratio >= 0.0 && std::isfinite(ratio)), "ratio must be >= 0 (NaN: no test)");
  P2P_REQUIRE(offsets0 && offsets1 && offsets0_host && offsets1_host, "null offsets");
  P2P_REQUIRE(offsets0_host[0] == 0 && offsets1_host[0] == 0, "offsets must start at 0");
  int max0 = 0, max1 = 0;
  for (int k = 0; k < n_pairs; ++k) {
    const int64_t a = offsets0_host[k + 1] - offsets0_host[k], b = offsets1_host[k + 1] - offsets1_host[k];
    P2P_REQUIRE(a >= 0 && a < (1 << 20) && b >= 0 && b < (1 << 20), "every set must hold 0 .. 2^20 - 1 descriptors");
    max0 = std::max(max0, (int)a);
    max1 = std::max(max1, (int)b);
  }
  const long long n0 = offsets0_host[n_pairs], n1 = offsets1_host[n_pairs];
  P2P_REQUIRE((d0 && match && sim) || n0 == 0, "null pointer");
  P2P_REQUIRE(d1 || n1 == 0, "null pointer");
  if (n0 == 0) return 0;
  return launch_match_descriptors(h->sp, d0, d1, (const long long*)offsets0, (const long long*)offsets1, n_pairs, dim,
                                  max0, max1, n0, n1, mutual, !std::isnan(min_sim), min_sim, !std::isnan(ratio), ratio,
                                  h->opt_match_impl, match, sim, tc_sim, tc_idx, eps, n_fixed,
                                  reinterpret_cast<cudaStream_t>(stream));
}

int p2p_sg_sinkhorn(p2p_handle_t h, const float* scores, int batch, int n, int m, const float* alpha, int iters,
                    float match_threshold, float* log_assign, int32_t* matches0, int32_t* matches1, float* mscores0,
                    float* mscores1, void* stream) {
  P2P_ENTER(h);
  P2P_REQUIRE(batch >= 1 && n >= 1 && m >= 1, "batch, n and m must be >= 1");
  P2P_REQUIRE(n <= kSgMaxPoints && m <= kSgMaxPoints, "n and m must be <= 2^20");
  P2P_REQUIRE((long long)batch * (n + 1) * (m + 1) < (1ll << 31), "batch * (n + 1) * (m + 1) must be < 2^31");
  P2P_REQUIRE(iters >= 0 && iters <= kSgMaxIters, "iters must be in 0..100000");
  P2P_REQUIRE(std::isfinite(match_threshold), "match_threshold must be finite");
  P2P_REQUIRE(scores && alpha, "null pointer");
  return launch_sg_sinkhorn(h->sg, scores, batch, n, m, alpha, iters, match_threshold, log_assign, matches0, matches1,
                            mscores0, mscores1, std::min(sms(h), h->num_sms), reinterpret_cast<cudaStream_t>(stream));
}

}  // extern "C"
