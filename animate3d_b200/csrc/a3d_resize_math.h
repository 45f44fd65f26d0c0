// Arithmetic of the CLIP image preprocessing, shared by the CUDA kernel (a3d_clip.cu) and by the CPU test harness
// (tests/cpu_harness/clip_resize_cpu.cpp).
//
// The contract is what the reference does to the frame-0 renders before the IP-Adapter image encoder
// (custom/threestudio-animate3d/guidance/animatemv_guidance.py:546-555, transformers 4.25-4.28 CLIP processor):
//   uint8 = trunc(fp32(x) * 255)                              ((x*255).astype(np.uint8) on the host copy)
//   resize so that the short edge is 224 and the long edge int(224 * long / short), with Pillow's Image.resize(BICUBIC):
//     a = -0.5, support 2 * max(scale, 1), weights in double normalised per output sample, then 22-bit fixed point with
//     +-0.5 rounding; horizontal pass first, then vertical; each pass rounds (+2^21) and clamps to uint8
//   centre crop 224 x 224 at top / left = floor((size - 224) / 2)
//   pixel = (fp32(u) / 255 - mean[c]) / std[c] in fp32 (OpenAI CLIP mean / std)
// The coefficient tables are built on the host (resize_window, fixed_coeff); the per-pixel functions are __host__ __device__.
#pragma once
#include <math.h>
#include <stdint.h>

#ifndef A3D_HD
#if defined(__CUDACC__)
#define A3D_HD __host__ __device__ __forceinline__
#else
#define A3D_HD inline
#endif
#endif

namespace a3d {

constexpr int kResizePrecisionBits = 22;   // Pillow's PRECISION_BITS for 8-bit images (32 - 8 - 2)
constexpr int kClipSize = 224;             // shortest edge and centre crop of the ViT-H/14 processor
constexpr int kClipPatch = 14;
constexpr int kClipGrid = kClipSize / kClipPatch;             // 16 patches per side
constexpr int kClipTokens = kClipGrid * kClipGrid + 1;        // 257: class token + 256 patches
constexpr int kClipPatchK = 3 * kClipPatch * kClipPatch;      // 588 = (c, ky, kx) of the flattened conv weight
constexpr int kClipPatchKPad = 640;                           // K of the patch GEMM: 588 zero-padded to a multiple of 64

// ---------------------------------------------------------------- host: shapes and coefficient tables
// CLIP resize target: the short edge becomes 224, the long edge int(224 * long / short) (Python float division).
inline void clip_resize_shape(int h, int w, int* rh, int* rw) {
  if (w <= h) {
    *rw = kClipSize;
    *rh = (int)((double)kClipSize * h / w);
  } else {
    *rh = kClipSize;
    *rw = (int)((double)kClipSize * w / h);
  }
}

inline double bicubic_filter(double x) {
  const double a = -0.5;
  if (x < 0.0) x = -x;
  if (x < 1.0) return ((a + 2.0) * x - (a + 3.0)) * x * x + 1.0;
  if (x < 2.0) return (((x - 5.0) * x + 8.0) * x - 4.0) * a;
  return 0.0;
}

// Taps per output sample of a resize in_size -> out_size (Pillow's ksize).
inline int resize_ksize(int in_size, int out_size) {
  double filterscale = (double)in_size / out_size;
  if (filterscale < 1.0) filterscale = 1.0;
  return (int)ceil(2.0 * filterscale) * 2 + 1;
}

// Pillow's precompute_coeffs: bounds[2 o] = first input sample, bounds[2 o + 1] = number of taps; w[o * ksize + i] the
// normalised double weights (0 past the taps).
inline void resize_window(int in_size, int out_size, int32_t* bounds, double* w) {
  const double scale = (double)in_size / out_size;
  const double filterscale = scale < 1.0 ? 1.0 : scale;
  const double support = 2.0 * filterscale;
  const int ksize = resize_ksize(in_size, out_size);
  const double ss = 1.0 / filterscale;
  for (int o = 0; o < out_size; ++o) {
    const double center = (o + 0.5) * scale;
    int xmin = (int)(center - support + 0.5);
    if (xmin < 0) xmin = 0;
    int xmax = (int)(center + support + 0.5);
    if (xmax > in_size) xmax = in_size;
    xmax -= xmin;
    double* k = w + (int64_t)o * ksize;
    double ww = 0.0;
    int x = 0;
    for (; x < xmax; ++x) {
      k[x] = bicubic_filter((x + xmin - center + 0.5) * ss);
      ww += k[x];
    }
    for (x = 0; x < xmax; ++x)
      if (ww != 0.0) k[x] /= ww;
    for (; x < ksize; ++x) k[x] = 0.0;
    bounds[2 * o] = xmin;
    bounds[2 * o + 1] = xmax;
  }
}

// Pillow's normalize_coeffs_8bpc: round half away from zero into 22-bit fixed point.
inline int32_t fixed_coeff(double w) {
  const double s = w * (double)(1 << kResizePrecisionBits);
  return w < 0 ? (int32_t)(-0.5 + s) : (int32_t)(0.5 + s);
}

// ---------------------------------------------------------------- per-pixel arithmetic (host and device)
// (x * 255).astype(np.uint8) on an fp32 x: truncation.  Outside [0, 1] (and NaN) numpy's cast is undefined; here it clamps.
A3D_HD uint8_t quantise_u8(float x) {
  const float v = x * 255.0f;
  if (!(v > 0.0f)) return 0;
  if (v >= 255.0f) return 255;
  return (uint8_t)(int)v;
}

// Pillow's clip8: the fixed-point sum (with its +2^21 rounding term) back to uint8.
A3D_HD uint8_t resize_clip8(int32_t ss) {
  if (ss <= 0) return 0;
  if (ss >= (256 << kResizePrecisionBits)) return 255;
  return (uint8_t)(ss >> kResizePrecisionBits);
}

// One output sample of one pass: sum over the n taps starting at input sample first, src(i) the uint8 at input index i.
template <class Src>
A3D_HD uint8_t resize_tap(const int32_t* k, int first, int n, const Src& src) {
  int32_t ss = 1 << (kResizePrecisionBits - 1);
  for (int i = 0; i < n; ++i) ss += (int32_t)src(first + i) * k[i];
  return resize_clip8(ss);
}

// Output pixel (oy, ox) of the resized image: the vertical pass over horizontal-pass rows, as Pillow's two passes compute it.
template <class Src>
A3D_HD uint8_t resize_pixel(int oy, int ox, const int32_t* bounds_y, const int32_t* coeffs_y, int ksize_y, const int32_t* bounds_x,
                            const int32_t* coeffs_x, int ksize_x, const Src& src) {
  const int32_t* kx = coeffs_x + (int64_t)ox * ksize_x;
  const int x0 = bounds_x[2 * ox], nx = bounds_x[2 * ox + 1];
  return resize_tap(coeffs_y + (int64_t)oy * ksize_y, bounds_y[2 * oy], bounds_y[2 * oy + 1],
                    [&](int iy) { return resize_tap(kx, x0, nx, [&](int ix) { return src(iy, ix); }); });
}

A3D_HD float clip_normalise(uint8_t u, int c) {
  const float mean = c == 0 ? 0.48145466f : (c == 1 ? 0.4578275f : 0.40821073f);
  const float stdv = c == 0 ? 0.26862954f : (c == 1 ? 0.26130258f : 0.27577711f);
  return ((float)u / 255.0f - mean) / stdv;
}

}  // namespace a3d
