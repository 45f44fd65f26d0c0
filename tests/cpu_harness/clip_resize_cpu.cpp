// CPU driver of the CLIP preprocessing arithmetic (animate3d_b200/csrc/a3d_resize_math.h), for tests/test_clip_cpu.py.
// `variant` selects deliberate faults for the negative controls: 0 = the contract, 1 = round the float input instead of
// truncating, 2 = vertical pass first, 3 = fixed-point coefficients without the +-0.5 rounding.
#include <math.h>
#include <stdint.h>

#include <vector>

#include "../../animate3d_b200/csrc/a3d_resize_math.h"

using namespace a3d;

namespace {

struct Tables {
  std::vector<int32_t> bounds, coeffs;
  int ksize;
};

Tables tables(int in_size, int out_size, int variant) {
  Tables t;
  t.ksize = resize_ksize(in_size, out_size);
  t.bounds.resize(2 * out_size);
  std::vector<double> w((size_t)out_size * t.ksize);
  resize_window(in_size, out_size, t.bounds.data(), w.data());
  t.coeffs.resize(w.size());
  for (size_t i = 0; i < w.size(); ++i)
    t.coeffs[i] = variant == 3 ? (int32_t)(w[i] * (double)(1 << kResizePrecisionBits)) : fixed_coeff(w[i]);
  return t;
}

// src(iy, ix) -> uint8 of one channel; out [oh, ow]
template <class Src>
void resize_channel(int h, int w, int oh, int ow, int variant, const Src& src, uint8_t* out) {
  const Tables ty = tables(h, oh, variant), tx = tables(w, ow, variant);
  for (int oy = 0; oy < oh; ++oy)
    for (int ox = 0; ox < ow; ++ox) {
      if (variant == 2) {
        const int32_t* ky = ty.coeffs.data() + (size_t)oy * ty.ksize;
        const int y0 = ty.bounds[2 * oy], ny = ty.bounds[2 * oy + 1];
        out[oy * ow + ox] = resize_tap(tx.coeffs.data() + (size_t)ox * tx.ksize, tx.bounds[2 * ox], tx.bounds[2 * ox + 1],
                                       [&](int ix) { return resize_tap(ky, y0, ny, [&](int iy) { return src(iy, ix); }); });
      } else {
        out[oy * ow + ox] = resize_pixel(oy, ox, ty.bounds.data(), ty.coeffs.data(), ty.ksize, tx.bounds.data(), tx.coeffs.data(),
                                         tx.ksize, src);
      }
    }
}

}  // namespace

extern "C" {

// Image.resize((ow, oh), BICUBIC) of a uint8 [h, w, 3] image -> out [oh, ow, 3]
void clip_resize_u8(const uint8_t* src, int h, int w, int oh, int ow, int variant, uint8_t* out) {
  std::vector<uint8_t> ch((size_t)oh * ow);
  for (int c = 0; c < 3; ++c) {
    resize_channel(h, w, oh, ow, variant, [&](int iy, int ix) { return src[((size_t)iy * w + ix) * 3 + c]; }, ch.data());
    for (size_t i = 0; i < ch.size(); ++i) out[i * 3 + c] = ch[i];
  }
}

// The processor on an fp32 [3, h, w] render in [0, 1]: u8 [3, 224, 224] after the crop, pixel_values [3, 224, 224]
void clip_prep_f32(const float* src, int h, int w, int variant, uint8_t* u8_out, float* pv_out) {
  int rh, rw;
  clip_resize_shape(h, w, &rh, &rw);
  std::vector<uint8_t> r((size_t)rh * rw);
  for (int c = 0; c < 3; ++c) {
    const float* s = src + (size_t)c * h * w;
    resize_channel(h, w, rh, rw, variant, [&](int iy, int ix) -> uint8_t {
      const float x = s[(size_t)iy * w + ix];
      if (variant == 1) {
        const float v = rintf(x * 255.0f);
        return (uint8_t)(v < 0.f ? 0.f : (v > 255.f ? 255.f : v));
      }
      return quantise_u8(x);
    }, r.data());
    const int top = (rh - kClipSize) / 2, left = (rw - kClipSize) / 2;
    for (int y = 0; y < kClipSize; ++y)
      for (int x = 0; x < kClipSize; ++x) {
        const uint8_t u = r[(size_t)(y + top) * rw + x + left];
        u8_out[((size_t)c * kClipSize + y) * kClipSize + x] = u;
        pv_out[((size_t)c * kClipSize + y) * kClipSize + x] = clip_normalise(u, c);
      }
  }
}

}  // extern "C"
