// Image preprocessing on the GPU: the tensor half of `load_im_flexible` (utils/datasets/preprocess.py:32-60):
//   transforms.functional.resize(img, (ht, wt), Image.BICUBIC)  ->  ToTensor  ->  Normalize(ImageNet mean / std)
// for an already decoded 8-bit RGB image (JPEG/PNG decoding stays host I/O).
//
// PIL is a third-party dependency of the reference (Pillow; environment.yml does not pin it, 12.2.0 is installed
// here).  Its 8-bit resampling is integer arithmetic and therefore reproducible BIT-EXACTLY; this file restates the
// published algorithm of Pillow's src/libImaging/Resample.c:
//   * precompute_coeffs: per output coordinate, centre = (xx + 0.5) * scale, support = 2 * max(scale, 1) (bicubic,
//     a = -0.5, antialiasing when down-scaling), window [xmin, xmax) clipped to the image, weights normalised to 1
//     (double precision, done on the host exactly as Pillow does);
//   * normalize_coeffs_8bpc: weights -> fixed point with PRECISION_BITS = 32 - 8 - 2 = 22, rounded half away from 0;
//   * ImagingResampleHorizontal_8bpc then ImagingResampleVertical_8bpc: int32 accumulation starting at
//     1 << (PRECISION_BITS - 1), result clip8(acc >> PRECISION_BITS); the horizontal result is rounded to uint8
//     before the vertical pass.
// ToTensor is float32(u8) / 255 and Normalize (x - mean) / std in float32 (torchvision), reproduced with
// correctly rounded IEEE operations.
// The optional grey image is Pillow's convert('L') of the (resized) 8-bit image, src/libImaging/Convert.c rgb2l:
// L = (19595 R + 38470 G + 7471 B + 0x8000) >> 16 (ITU-R 601-2 luma in 16-bit fixed point), then ToTensor's / 255.
#include <math.h>

#include <vector>

#include "kernels.h"

namespace p2p {

constexpr int kPrecBits = 32 - 8 - 2;

static double bicubic_filter(double x) {
  const double a = -0.5;
  if (x < 0.0) x = -x;
  if (x < 1.0) return ((a + 2.0) * x - (a + 3.0)) * x * x + 1;
  if (x < 2.0) return (((x - 5) * x + 8) * x - 4) * a;
  return 0.0;
}

// Pillow's precompute_coeffs + normalize_coeffs_8bpc for one axis (box = the whole image).
int resample_coeffs(int in_size, int out_size, std::vector<int>& bounds, std::vector<int>& kk) {
  const double scale = (double)in_size / out_size;
  double filterscale = scale;
  if (filterscale < 1.0) filterscale = 1.0;
  const double support = 2.0 * filterscale;
  const int ksize = (int)ceil(support) * 2 + 1;
  bounds.assign((size_t)out_size * 2, 0);
  kk.assign((size_t)out_size * ksize, 0);
  std::vector<double> k(ksize);
  for (int xx = 0; xx < out_size; ++xx) {
    const double center = (xx + 0.5) * scale;
    double ww = 0.0;
    const double ss = 1.0 / filterscale;
    int xmin = (int)(center - support + 0.5);
    if (xmin < 0) xmin = 0;
    int xmax = (int)(center + support + 0.5);
    if (xmax > in_size) xmax = in_size;
    xmax -= xmin;
    int x = 0;
    for (; x < xmax; ++x) {
      const double w = bicubic_filter((x + xmin - center + 0.5) * ss);
      k[x] = w;
      ww += w;
    }
    for (x = 0; x < xmax; ++x)
      if (ww != 0.0) k[x] /= ww;
    for (; x < ksize; ++x) k[x] = 0;
    bounds[xx * 2 + 0] = xmin;
    bounds[xx * 2 + 1] = xmax;
    for (x = 0; x < ksize; ++x)
      kk[(size_t)xx * ksize + x] = k[x] < 0 ? (int)(-0.5 + k[x] * (1 << kPrecBits)) : (int)(0.5 + k[x] * (1 << kPrecBits));
  }
  return ksize;
}

__device__ __forceinline__ uint8_t clip8(int v) {
  v >>= kPrecBits;        // arithmetic shift, as Pillow's lookup table index
  return (uint8_t)(v < 0 ? 0 : (v > 255 ? 255 : v));
}

// horizontal pass: in [H][Win][3] u8 -> tmp [H][Wout][3] u8
__global__ void resample_h_kernel(const uint8_t* __restrict__ in, int H, int Win, int Wout, const int* __restrict__ bounds,
                                  const int* __restrict__ kk, int ksize, uint8_t* __restrict__ tmp) {
  const int xx = blockIdx.x * blockDim.x + threadIdx.x, yy = blockIdx.y;
  if (xx >= Wout) return;
  const int xmin = bounds[xx * 2], xmax = bounds[xx * 2 + 1];
  const int* k = kk + (size_t)xx * ksize;
  int s0 = 1 << (kPrecBits - 1), s1 = s0, s2 = s0;
  const uint8_t* row = in + ((size_t)yy * Win + xmin) * 3;
  for (int x = 0; x < xmax; ++x) {
    const int w = k[x];
    s0 += row[x * 3 + 0] * w;
    s1 += row[x * 3 + 1] * w;
    s2 += row[x * 3 + 2] * w;
  }
  uint8_t* o = tmp + ((size_t)yy * Wout + xx) * 3;
  o[0] = clip8(s0);
  o[1] = clip8(s1);
  o[2] = clip8(s2);
}

// vertical pass + ToTensor + Normalize: tmp [Hin][W][3] u8 -> out [3][Hout][W] f32 and (optional) gray [Hout][W] f32.
// kk == nullptr: no resampling.
__global__ void resample_v_norm_kernel(const uint8_t* __restrict__ tmp, int Hin, int W, int Hout, const int* __restrict__ bounds,
                                       const int* __restrict__ kk, int ksize, float m0, float m1, float m2, float d0, float d1,
                                       float d2, float* __restrict__ out, uint8_t* __restrict__ out_u8,
                                       float* __restrict__ gray) {
  const int xx = blockIdx.x * blockDim.x + threadIdx.x, yy = blockIdx.y;
  if (xx >= W) return;
  uint8_t px[3];
  if (kk != nullptr) {
    const int ymin = bounds[yy * 2], ymax = bounds[yy * 2 + 1];
    const int* k = kk + (size_t)yy * ksize;
    int s0 = 1 << (kPrecBits - 1), s1 = s0, s2 = s0;
    for (int y = 0; y < ymax; ++y) {
      const uint8_t* p = tmp + ((size_t)(y + ymin) * W + xx) * 3;
      const int w = k[y];
      s0 += p[0] * w;
      s1 += p[1] * w;
      s2 += p[2] * w;
    }
    px[0] = clip8(s0);
    px[1] = clip8(s1);
    px[2] = clip8(s2);
  } else {
    const uint8_t* p = tmp + ((size_t)yy * W + xx) * 3;
    px[0] = p[0];
    px[1] = p[1];
    px[2] = p[2];
  }
  const size_t plane = (size_t)Hout * W, o = (size_t)yy * W + xx;
  if (out_u8 != nullptr) {
    out_u8[o * 3 + 0] = px[0];
    out_u8[o * 3 + 1] = px[1];
    out_u8[o * 3 + 2] = px[2];
  }
  out[o] = __fdiv_rn(__fsub_rn(__fdiv_rn((float)px[0], 255.f), m0), d0);
  out[plane + o] = __fdiv_rn(__fsub_rn(__fdiv_rn((float)px[1], 255.f), m1), d1);
  out[2 * plane + o] = __fdiv_rn(__fsub_rn(__fdiv_rn((float)px[2], 255.f), m2), d2);
  if (gray != nullptr) {
    const int l = (px[0] * 19595 + px[1] * 38470 + px[2] * 7471 + 0x8000) >> 16;
    gray[o] = __fdiv_rn((float)l, 255.f);
  }
}

// Coefficient tables of one (ho, wo) -> (ht, wt) geometry, uploaded once (synchronously) and cached by the handle.
int preprocess_build_coefs(int ho, int wo, int ht, int wt, PreprocessCoefs& C) {
  std::vector<int> bx, kx, by, ky;
  C.ho = ho; C.wo = wo; C.ht = ht; C.wt = wt;
  C.ksx = wt != wo ? resample_coeffs(wo, wt, bx, kx) : 0;
  C.ksy = ht != ho ? resample_coeffs(ho, ht, by, ky) : 0;
  std::vector<int> all;
  C.o_bx = all.size(); all.insert(all.end(), bx.begin(), bx.end());
  C.o_kx = all.size(); all.insert(all.end(), kx.begin(), kx.end());
  C.o_by = all.size(); all.insert(all.end(), by.begin(), by.end());
  C.o_ky = all.size(); all.insert(all.end(), ky.begin(), ky.end());
  C.d = nullptr;
  if (!all.empty()) {
    P2P_CUDA_OK(cudaMalloc(&C.d, all.size() * sizeof(int)));
    P2P_CUDA_OK(cudaMemcpy(C.d, all.data(), all.size() * sizeof(int), cudaMemcpyHostToDevice));
  }
  return 0;
}

// rgb: DEVICE u8 [ho][wo][3]; out: DEVICE f32 [3][ht][wt]; resized_u8 (optional): DEVICE u8 [ht][wt][3];
// gray (optional): DEVICE f32 [ht][wt]; tmp: DEVICE scratch of ho*wt*3 bytes (horizontal-pass result).
int launch_preprocess(const uint8_t* rgb, const PreprocessCoefs& C, const float mean[3], const float stdv[3], float* out,
                      uint8_t* resized_u8, float* gray, uint8_t* tmp, cudaStream_t st) {
  const int ho = C.ho, wo = C.wo, ht = C.ht, wt = C.wt;
  const uint8_t* src = rgb;
  if (C.ksx > 0) {
    dim3 grid(cdiv(wt, 128), ho);
    resample_h_kernel<<<grid, 128, 0, st>>>(rgb, ho, wo, wt, C.d + C.o_bx, C.d + C.o_kx, C.ksx, tmp);
    P2P_LAUNCH_OK();
    src = tmp;
  }
  dim3 grid(cdiv(wt, 128), ht);
  resample_v_norm_kernel<<<grid, 128, 0, st>>>(src, ho, wt, ht, C.ksy > 0 ? C.d + C.o_by : nullptr,
                                               C.ksy > 0 ? C.d + C.o_ky : nullptr, C.ksy, mean[0], mean[1], mean[2], stdv[0],
                                               stdv[1], stdv[2], out, resized_u8, gray);
  P2P_LAUNCH_OK();
  return 0;
}

}  // namespace p2p
