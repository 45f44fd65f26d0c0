// CLIP image preprocessing of the IP-Adapter image encoder (ViT-H/14), straight into the A operand of the patch-embedding
// GEMM: uint8 quantisation, Pillow-exact bicubic resize, centre crop, normalisation and patchify in one launch.  The
// arithmetic lives in a3d_resize_math.h (shared with the CPU harness); the resize coefficient tables are built on the host.
// Replaces the host round trip at custom/threestudio-animate3d/guidance/animatemv_guidance.py:546-555 (.cpu() -> PIL ->
// CLIPImageProcessor) and the patch-embedding convolution of transformers' CLIPVisionEmbeddings.
#include "a3d_common.cuh"
#include "a3d_host.cuh"
#include "a3d_resize_math.h"

namespace a3d {

struct ClipPrepDev {
  const void* src;
  int fmt, h, w;
  const int32_t *bx, *cx, *by, *cy;
  int kx, ky;
  int crop_x, crop_y;
  __half* patches;
  float* pixels;
};

// One thread per element of the patch-GEMM A operand [n * 257, 640]: row 0 of an image (the class token, which comes from
// the GEMM's row-bias table) and the K padding 588..639 are zero; column k = (c, ky, kx) of patch row r reads pixel
// (c, 14 (r - 1) / 16 + ky, 14 (r - 1) % 16 + kx) of the 224 x 224 crop.  Every crop pixel is visited exactly once, so the
// same thread also writes pixel_values when asked.
__global__ void clip_preprocess_kernel(const ClipPrepDev p, int64_t total) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int64_t row = idx / kClipPatchKPad;
  const int k = (int)(idx % kClipPatchKPad);
  const int img = (int)(row / kClipTokens), tok = (int)(row % kClipTokens);
  if (tok == 0 || k >= kClipPatchK) {
    if (p.patches) p.patches[idx] = __float2half_rn(0.f);
    return;
  }
  const int c = k / (kClipPatch * kClipPatch);
  const int y = ((tok - 1) / kClipGrid) * kClipPatch + (k / kClipPatch) % kClipPatch;
  const int x = ((tok - 1) % kClipGrid) * kClipPatch + k % kClipPatch;
  float v;
  if (p.fmt == A3D_CLIP_SRC_PIXELS) {
    v = reinterpret_cast<const float*>(p.src)[(((int64_t)img * 3 + c) * kClipSize + y) * kClipSize + x];
  } else {
    uint8_t u;
    if (p.fmt == A3D_CLIP_SRC_F32_NCHW) {
      const float* s = reinterpret_cast<const float*>(p.src) + ((int64_t)img * 3 + c) * p.h * p.w;
      u = resize_pixel(y + p.crop_y, x + p.crop_x, p.by, p.cy, p.ky, p.bx, p.cx, p.kx,
                       [&](int iy, int ix) { return quantise_u8(__ldg(s + (int64_t)iy * p.w + ix)); });
    } else {
      const uint8_t* s = reinterpret_cast<const uint8_t*>(p.src) + (int64_t)img * p.h * p.w * 3 + c;
      u = resize_pixel(y + p.crop_y, x + p.crop_x, p.by, p.cy, p.ky, p.bx, p.cx, p.kx,
                       [&](int iy, int ix) { return __ldg(s + ((int64_t)iy * p.w + ix) * 3); });
    }
    v = clip_normalise(u, c);
    if (p.pixels) p.pixels[(((int64_t)img * 3 + c) * kClipSize + y) * kClipSize + x] = v;
  }
  if (p.patches) p.patches[idx] = __float2half_rn(v);
}

}  // namespace a3d

extern "C" int a3d_clip_resize_plan(int h, int w, int* resize_h, int* resize_w, int* ksize_y, int* ksize_x) {
  using namespace a3d;
  if (h <= 0 || w <= 0 || !resize_h || !resize_w || !ksize_y || !ksize_x)
    return fail(A3D_EINVAL, "a3d_clip_resize_plan: bad image size %d x %d", h, w);
  clip_resize_shape(h, w, resize_h, resize_w);
  *ksize_y = resize_ksize(h, *resize_h);
  *ksize_x = resize_ksize(w, *resize_w);
  return A3D_OK;
}

extern "C" int a3d_clip_resize_coeffs(int in_size, int out_size, int32_t* bounds_host, int32_t* coeffs_host) {
  using namespace a3d;
  if (in_size <= 0 || out_size <= 0 || !bounds_host || !coeffs_host)
    return fail(A3D_EINVAL, "a3d_clip_resize_coeffs: bad sizes %d -> %d", in_size, out_size);
  const int ksize = resize_ksize(in_size, out_size);
  double* w = new double[(size_t)out_size * ksize];
  resize_window(in_size, out_size, bounds_host, w);
  for (int64_t i = 0; i < (int64_t)out_size * ksize; ++i) coeffs_host[i] = fixed_coeff(w[i]);
  delete[] w;
  return A3D_OK;
}

extern "C" int a3d_clip_preprocess(const a3d_clip_prep_args* a, void* stream) {
  using namespace a3d;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (!a || !a->src || a->n <= 0 || (!a->patches && !a->pixel_values))
    return fail(A3D_EINVAL, "a3d_clip_preprocess: null operand or no output");
  ClipPrepDev d;
  memset(&d, 0, sizeof(d));
  d.src = a->src; d.fmt = a->src_format;
  d.patches = reinterpret_cast<__half*>(a->patches);
  if (a->src_format == A3D_CLIP_SRC_PIXELS) {
    if (!a->patches) return fail(A3D_EINVAL, "a3d_clip_preprocess: pixel input needs the patch output");
  } else if (a->src_format == A3D_CLIP_SRC_F32_NCHW || a->src_format == A3D_CLIP_SRC_U8_NHWC) {
    int rh, rw, ky, kx;
    if (int r = a3d_clip_resize_plan(a->h, a->w, &rh, &rw, &ky, &kx)) return r;
    if (rh != a->resize_h || rw != a->resize_w || ky != a->ksize_y || kx != a->ksize_x)
      return fail(A3D_EINVAL, "a3d_clip_preprocess: tables for %d x %d (k %d, %d) do not match the plan of a %d x %d image "
                  "(%d x %d, k %d, %d)", a->resize_h, a->resize_w, a->ksize_y, a->ksize_x, a->h, a->w, rh, rw, ky, kx);
    if (!a->bounds_x || !a->coeffs_x || !a->bounds_y || !a->coeffs_y)
      return fail(A3D_EINVAL, "a3d_clip_preprocess: missing resize tables");
    d.h = a->h; d.w = a->w;
    d.bx = a->bounds_x; d.cx = a->coeffs_x; d.kx = kx;
    d.by = a->bounds_y; d.cy = a->coeffs_y; d.ky = ky;
    d.crop_x = (rw - kClipSize) / 2; d.crop_y = (rh - kClipSize) / 2;
    d.pixels = a->pixel_values;
  } else {
    return fail(A3D_EINVAL, "a3d_clip_preprocess: unknown source format %d", a->src_format);
  }
  // with pixel_values only, the kernel still walks the A-operand index space (each crop pixel once) and skips the fp16 stores
  const int64_t total = (int64_t)a->n * kClipTokens * kClipPatchKPad;
  clip_preprocess_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(d, total);
  A3D_LAUNCH_CHECK();
  return A3D_OK;
}
