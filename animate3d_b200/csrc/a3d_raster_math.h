// Per-gaussian and per-(pixel,gaussian) arithmetic of the splat rasterizer, shared by the CUDA kernels (a3d_raster*.cu)
// and by the CPU test harness (tests/cpu_harness/raster_cpu.cpp) -- every function is __host__ __device__.
//
// Restates the algorithm of graphdeco-inria/diff-gaussian-rasterization + ashawkey's depth/alpha fork (the un-vendored
// dependency the reference calls at custom/threestudio-animate3d/renderer/diff_gaussian_rasterizer_advanced_4d.py:161-170),
// as recorded in SURVEY.md Appendix C.  The floating-point operation order of the FORWARD preprocess is the one written
// in oracle/raster_oracle.py::preprocess: translation units that include this header for the preprocess are compiled
// with --fmad=false so radii, tile rectangles and depth keys agree bit for bit with the oracle.
#pragma once
#include <math.h>
#include <stdint.h>

#if defined(__CUDACC__)
#define A3D_HD __host__ __device__ __forceinline__
#else
#define A3D_HD inline
#endif

namespace a3d {

constexpr int kTile = 16;
constexpr float kShC0 = 0.28209479177387814f;

struct PreGauss {
  float depth;
  int radius;
  float px, py;
  float conA, conB, conC;
  float cov3[6];
  int rx0, ry0, rx1, ry1;
  int tiles;
};

A3D_HD void quat_to_rot(const float* q, float R[9]) {
  const float r = q[0], x = q[1], y = q[2], z = q[3];
  R[0] = 1.0f - 2.0f * (y * y + z * z); R[1] = 2.0f * (x * y - r * z); R[2] = 2.0f * (x * z + r * y);
  R[3] = 2.0f * (x * y + r * z); R[4] = 1.0f - 2.0f * (x * x + z * z); R[5] = 2.0f * (y * z - r * x);
  R[6] = 2.0f * (x * z - r * y); R[7] = 2.0f * (y * z + r * x); R[8] = 1.0f - 2.0f * (x * x + y * y);
}

A3D_HD void cov3d_from_scale_rot(const float* s_in, float mod, const float* q, float cov[6]) {
  float R[9];
  quat_to_rot(q, R);
  const float s[3] = {s_in[0] * mod, s_in[1] * mod, s_in[2] * mod};
  float M[9];
  for (int i = 0; i < 3; ++i)
    for (int k = 0; k < 3; ++k) M[i * 3 + k] = R[i * 3 + k] * s[k];
  auto dot = [&](int i, int j) { return (M[i * 3] * M[j * 3] + M[i * 3 + 1] * M[j * 3 + 1]) + M[i * 3 + 2] * M[j * 3 + 2]; };
  cov[0] = dot(0, 0); cov[1] = dot(0, 1); cov[2] = dot(0, 2); cov[3] = dot(1, 1); cov[4] = dot(1, 2); cov[5] = dot(2, 2);
}

A3D_HD int clamp_trunc(float v, int hi) {
  int i = (int)v;  // truncation toward zero, like the (int) cast upstream
  if (!(v == v)) i = 0;
  if (v >= 1e9f) i = hi;
  if (v <= -1e9f) i = 0;
  return i < 0 ? 0 : (i > hi ? hi : i);
}

// Forward preprocess of one gaussian (SURVEY C.1).  Returns false (tiles = 0, radius = 0) when culled.
A3D_HD bool preprocess_gaussian(const float* p, const float* s, const float* q, float mod, const float* vm, const float* pm,
                                float tanfovx, float tanfovy, int H, int W, PreGauss& o) {
  const float px = p[0], py = p[1], pz = p[2];
  auto tp = [&](const float* m, int c) { return ((m[c] * px + m[4 + c] * py) + m[8 + c] * pz) + m[12 + c]; };
  const float tx = tp(vm, 0), ty = tp(vm, 1), tz = tp(vm, 2);
  o.depth = tz; o.radius = 0; o.tiles = 0;
  o.rx0 = o.ry0 = o.rx1 = o.ry1 = 0;
  const float hx = tp(pm, 0), hy = tp(pm, 1), hw = tp(pm, 3);
  const float p_w = 1.0f / (hw + 1e-7f);
  const float projx = hx * p_w, projy = hy * p_w;
  o.px = ((projx + 1.0f) * (float)W - 1.0f) * 0.5f;
  o.py = ((projy + 1.0f) * (float)H - 1.0f) * 0.5f;
  o.conA = o.conB = o.conC = 0.f;
  cov3d_from_scale_rot(s, mod, q, o.cov3);
  if (!(tz > 0.2f)) return false;
  const float focal_x = (float)W / (2.0f * tanfovx), focal_y = (float)H / (2.0f * tanfovy);
  const float limx = 1.3f * tanfovx, limy = 1.3f * tanfovy;
  const float txc = fminf(limx, fmaxf(-limx, tx / tz)) * tz;
  const float tyc = fminf(limy, fmaxf(-limy, ty / tz)) * tz;
  const float j00 = focal_x / tz, j02 = -(focal_x * txc) / (tz * tz);
  const float j11 = focal_y / tz, j12 = -(focal_y * tyc) / (tz * tz);
  float m0[3], m1[3];
  for (int k = 0; k < 3; ++k) {
    m0[k] = j00 * vm[4 * k + 0] + j02 * vm[4 * k + 2];
    m1[k] = j11 * vm[4 * k + 1] + j12 * vm[4 * k + 2];
  }
  const float* c = o.cov3;
  const float S[3][3] = {{c[0], c[1], c[2]}, {c[1], c[3], c[4]}, {c[2], c[4], c[5]}};
  float v0[3], v1[3];
  for (int k = 0; k < 3; ++k) {
    v0[k] = (S[k][0] * m0[0] + S[k][1] * m0[1]) + S[k][2] * m0[2];
    v1[k] = (S[k][0] * m1[0] + S[k][1] * m1[1]) + S[k][2] * m1[2];
  }
  const float a = ((m0[0] * v0[0] + m0[1] * v0[1]) + m0[2] * v0[2]) + 0.3f;
  const float b = (m0[0] * v1[0] + m0[1] * v1[1]) + m0[2] * v1[2];
  const float cc = ((m1[0] * v1[0] + m1[1] * v1[1]) + m1[2] * v1[2]) + 0.3f;
  const float det = a * cc - b * b;
  if (det == 0.0f) return false;
  const float det_inv = 1.0f / det;
  o.conA = cc * det_inv; o.conB = -b * det_inv; o.conC = a * det_inv;
  const float mid = 0.5f * (a + cc);
  const float disc = sqrtf(fmaxf(mid * mid - det, 0.1f));
  const float lam = fmaxf(mid + disc, mid - disc);
  const float radius = ceilf(3.0f * sqrtf(lam));
  const int gx = (W + kTile - 1) / kTile, gy = (H + kTile - 1) / kTile;
  o.rx0 = clamp_trunc((o.px - radius) / (float)kTile, gx);
  o.rx1 = clamp_trunc((o.px + radius + (float)(kTile - 1)) / (float)kTile, gx);
  o.ry0 = clamp_trunc((o.py - radius) / (float)kTile, gy);
  o.ry1 = clamp_trunc((o.py + radius + (float)(kTile - 1)) / (float)kTile, gy);
  const int area = (o.rx1 - o.rx0) * (o.ry1 - o.ry0);
  if (area <= 0) return false;
  o.radius = (int)radius;
  o.tiles = area;
  return true;
}

// ---------------------------------------------------------------------------------------------------------------
// SH colour: rgb_ch = max(sum_k basis_k(dir) * sh_k,ch + 0.5, 0), dir = (mean - campos) / |mean - campos|
// ---------------------------------------------------------------------------------------------------------------
constexpr float kShC1 = 0.4886025119029199f;
// scalar constants: constexpr arrays are not usable in device code
constexpr float kShC2_0 = 1.0925484305920792f, kShC2_1 = -1.0925484305920792f, kShC2_2 = 0.31539156525252005f,
                kShC2_3 = -1.0925484305920792f, kShC2_4 = 0.5462742152960396f;
constexpr float kShC3_0 = -0.5900435899266435f, kShC3_1 = 2.890611442640554f, kShC3_2 = -0.4570457994644658f,
                kShC3_3 = 0.3731763325901154f, kShC3_4 = -0.4570457994644658f, kShC3_5 = 1.445305721320277f,
                kShC3_6 = -0.5900435899266435f;

A3D_HD void sh_basis(int deg, float x, float y, float z, float* b) {
  b[0] = kShC0;
  if (deg > 0) {
    b[1] = -kShC1 * y; b[2] = kShC1 * z; b[3] = -kShC1 * x;
    if (deg > 1) {
      const float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
      b[4] = kShC2_0 * xy; b[5] = kShC2_1 * yz; b[6] = kShC2_2 * (2.0f * zz - xx - yy);
      b[7] = kShC2_3 * xz; b[8] = kShC2_4 * (xx - yy);
      if (deg > 2) {
        b[9] = kShC3_0 * y * (3.0f * xx - yy); b[10] = kShC3_1 * xy * z;
        b[11] = kShC3_2 * y * (4.0f * zz - xx - yy); b[12] = kShC3_3 * z * (2.0f * zz - 3.0f * xx - 3.0f * yy);
        b[13] = kShC3_4 * x * (4.0f * zz - xx - yy); b[14] = kShC3_5 * z * (xx - yy);
        b[15] = kShC3_6 * x * (xx - 3.0f * yy);
      }
    }
  }
}

// unit direction from the camera centre to the gaussian mean m: the direction the SH colour is evaluated in; returns |m - campos|
A3D_HD float view_dir(const float* m, const float* campos, float& dx, float& dy, float& dz) {
  dx = m[0] - campos[0]; dy = m[1] - campos[1]; dz = m[2] - campos[2];
  const float n = sqrtf((dx * dx + dy * dy) + dz * dz);
  dx /= n; dy /= n; dz /= n;
  return n;
}

// forward colour of one (camera, gaussian) from its SH coefficients sh [(deg+1)^2][3]; bit ch of the result is set when
// channel ch was clamped at 0
A3D_HD uint32_t sh_colour(int deg, const float* m, const float* campos, const float* sh, float rgb[3]) {
  float dx, dy, dz, b[16];
  view_dir(m, campos, dx, dy, dz);
  sh_basis(deg, dx, dy, dz, b);
  const int nb = (deg + 1) * (deg + 1);
  uint32_t clamped = 0;
  for (int ch = 0; ch < 3; ++ch) {
    float v = 0.f;
    for (int k = 0; k < nb; ++k) v += b[k] * sh[3 * k + ch];
    v += 0.5f;
    if (v < 0.f) { clamped |= 1u << ch; v = 0.f; }
    rgb[ch] = v;
  }
  return clamped;
}

// Backward of sh_colour for one (camera, gaussian).  In: g = dL/drgb.  Out: g masked by the clamp bits, the basis b (so
// dL/dsh_k,ch = b[k] * g[ch]), and dL/dmean through the view direction ADDED to dmean.  The colour depends on the mean
// through dir even when the coefficients are frozen, so this term is needed whenever the mean gradient is.
A3D_HD void sh_backward(int deg, const float* m, const float* campos, const float* sh, uint32_t clamped, float g[3], float b[16],
                        float dmean[3]) {
  for (int ch = 0; ch < 3; ++ch)
    if (clamped & (1u << ch)) g[ch] = 0.f;
  float x, y, z;
  const float n = view_dir(m, campos, x, y, z);
  sh_basis(deg, x, y, z, b);
  if (deg == 0) return;
  // s_k = dL/dbasis_k; then dL/ddir = sum_k s_k * grad(basis_k)
  float s[16];
  const int nb = (deg + 1) * (deg + 1);
#pragma unroll
  for (int k = 1; k < 16; ++k) s[k] = k < nb ? (sh[3 * k] * g[0] + sh[3 * k + 1] * g[1]) + sh[3 * k + 2] * g[2] : 0.f;
  float gx = -kShC1 * s[3], gy = -kShC1 * s[1], gz = kShC1 * s[2];
  if (deg > 1) {
    const float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
    gx += kShC2_0 * y * s[4] - 2.f * kShC2_2 * x * s[6] + kShC2_3 * z * s[7] + 2.f * kShC2_4 * x * s[8];
    gy += kShC2_0 * x * s[4] + kShC2_1 * z * s[5] - 2.f * kShC2_2 * y * s[6] - 2.f * kShC2_4 * y * s[8];
    gz += kShC2_1 * y * s[5] + 4.f * kShC2_2 * z * s[6] + kShC2_3 * x * s[7];
    if (deg > 2) {
      gx += kShC3_0 * 6.f * xy * s[9] + kShC3_1 * yz * s[10] - kShC3_2 * 2.f * xy * s[11] - kShC3_3 * 6.f * xz * s[12] +
            kShC3_4 * (4.f * zz - 3.f * xx - yy) * s[13] + kShC3_5 * 2.f * xz * s[14] + kShC3_6 * 3.f * (xx - yy) * s[15];
      gy += kShC3_0 * 3.f * (xx - yy) * s[9] + kShC3_1 * xz * s[10] + kShC3_2 * (4.f * zz - xx - 3.f * yy) * s[11] -
            kShC3_3 * 6.f * yz * s[12] - kShC3_4 * 2.f * xy * s[13] - kShC3_5 * 2.f * yz * s[14] - kShC3_6 * 6.f * xy * s[15];
      gz += kShC3_1 * xy * s[10] + kShC3_2 * 8.f * yz * s[11] + kShC3_3 * (6.f * zz - 3.f * xx - 3.f * yy) * s[12] +
            kShC3_4 * 8.f * xz * s[13] + kShC3_5 * (xx - yy) * s[14];
    }
  }
  // dir = d / |d|: dL/dd = (I - dir dir^T) dL/ddir / |d|
  const float dot = (x * gx + y * gy) + z * gz;
  dmean[0] += (gx - x * dot) / n;
  dmean[1] += (gy - y * dot) / n;
  dmean[2] += (gz - z * dot) / n;
}

// ---------------------------------------------------------------------------------------------------------------
// blending: one (pixel, gaussian) step, forward and backward
// ---------------------------------------------------------------------------------------------------------------
// returns alpha (0 when the gaussian does not contribute)
A3D_HD float splat_alpha(float gx, float gy, float conA, float conB, float conC, float opac, float pixx, float pixy,
                         float* G_out) {
  const float dx = gx - pixx, dy = gy - pixy;
  const float power = -0.5f * (conA * dx * dx + conC * dy * dy) - conB * dx * dy;
  if (power > 0.0f) return 0.0f;
  const float G = expf(power);
  if (G_out) *G_out = G;
  const float alpha = fminf(0.99f, opac * G);
  if (alpha < 1.0f / 255.0f) return 0.0f;
  return alpha;
}

// ---------------------------------------------------------------------------------------------------------------
// RGBA8 test renders: the reference saves cat(render.clamp(0, 1), mask) as (rgba * 255).astype(np.uint8)
// (diff_gaussian_rasterizer_advanced_4d.py:180, systems/animate3d.py:439-445)
// ---------------------------------------------------------------------------------------------------------------
A3D_HD float clamp01(float v) { return fminf(fmaxf(v, 0.0f), 1.0f); }

// One rounded fp32 multiply by 255 (never contracted into an FMA), then numpy's float32 -> uint8 cast on x86: truncation
// toward zero to int32 and the low 8 bits of that (so 1.5 -> 126, -0.5 -> 129).  Defined for |v * 255| < 2^31.
A3D_HD uint8_t quantise_u8(float v) {
#if defined(__CUDA_ARCH__)
  const float p = __fmul_rn(v, 255.0f);
#else
  const float p = v * 255.0f;
#endif
  return (uint8_t)(uint32_t)(int32_t)p;
}

struct SplatGrad {   // partial derivatives of the loss w.r.t. one gaussian's screen-space quantities from ONE pixel
  float dmx, dmy;          // d/d(mean2D in pixels)
  float dconA, dconB, dconC;
  float dopac;
  float dcol[3];
  float ddepth;
};

// Backward step for a contributing gaussian (alpha > 0, T = transmittance BEFORE this gaussian).
// accum_* hold sum over gaussians BEHIND this one of (w_k * value_k) / T_after_this, maintained by the caller through
// the recurrences below (same as upstream's accum_rec / last_alpha / last_color).
A3D_HD void splat_backward(float gx, float gy, float conA, float conB, float conC, float opac, float pixx, float pixy,
                           float alpha, float G, float T, float T_final, const float col[3], float depth,
                           const float dL_dC[3], float dL_dD, float dL_dA, const float bg[3],
                           float accum_col[3], float& accum_depth, float& accum_alpha, float& last_alpha, float last_col[3],
                           float& last_depth, SplatGrad& g) {
  const float dx = gx - pixx, dy = gy - pixy;
  const float w = alpha * T;   // blending weight of this gaussian
  float dL_dalpha = 0.f;
  for (int ch = 0; ch < 3; ++ch) {
    accum_col[ch] = last_alpha * last_col[ch] + (1.f - last_alpha) * accum_col[ch];
    last_col[ch] = col[ch];
    dL_dalpha += (col[ch] - accum_col[ch]) * dL_dC[ch];
    g.dcol[ch] = w * dL_dC[ch];
  }
  accum_depth = last_alpha * last_depth + (1.f - last_alpha) * accum_depth;
  last_depth = depth;
  dL_dalpha += (depth - accum_depth) * dL_dD;
  g.ddepth = w * dL_dD;
  accum_alpha = last_alpha * 1.0f + (1.f - last_alpha) * accum_alpha;
  dL_dalpha += (1.0f - accum_alpha) * dL_dA;
  dL_dalpha *= T;
  last_alpha = alpha;
  float bg_dot = 0.f;
  for (int ch = 0; ch < 3; ++ch) bg_dot += bg[ch] * dL_dC[ch];
  dL_dalpha += (-T_final / (1.f - alpha)) * bg_dot;
  // alpha = min(0.99, opac * G): the clamp is treated as pass-through (upstream behaviour)
  const float dL_dG = opac * dL_dalpha;
  g.dopac = G * dL_dalpha;
  const float gdx = G * dx, gdy = G * dy;
  // dG/d(mean) = G * d(power)/d(mean), power = -0.5(A dx^2 + C dy^2) - B dx dy
  g.dmx = dL_dG * (-gdx * conA - gdy * conB);
  g.dmy = dL_dG * (-gdy * conC - gdx * conB);
  g.dconA = -0.5f * gdx * dx * dL_dG;
  g.dconB = -gdx * dy * dL_dG;
  g.dconC = -0.5f * gdy * dy * dL_dG;
}

// ---------------------------------------------------------------------------------------------------------------
// backward of the per-gaussian preprocess: (dconic, dmean2D[pixels], ddepth) -> (dmean3D, dscale, drot)
// ---------------------------------------------------------------------------------------------------------------
A3D_HD void preprocess_backward(const float* p, const float* s_in, const float* q, float mod, const float* vm, const float* pm,
                                float tanfovx, float tanfovy, int H, int W, float gA, float gB, float gC, float gpx, float gpy,
                                float gdepth, float dmean[3], float dscale[3], float drot[4]) {
  const float px = p[0], py = p[1], pz = p[2];
  auto tp = [&](const float* m, int c) { return ((m[c] * px + m[4 + c] * py) + m[8 + c] * pz) + m[12 + c]; };
  const float tx = tp(vm, 0), ty = tp(vm, 1), tz = tp(vm, 2);
  const float focal_x = (float)W / (2.0f * tanfovx), focal_y = (float)H / (2.0f * tanfovy);
  const float limx = 1.3f * tanfovx, limy = 1.3f * tanfovy;
  const float rx = tx / tz, ry = ty / tz;
  const bool clx = (rx < -limx) || (rx > limx), cly = (ry < -limy) || (ry > limy);
  const float cxr = fminf(limx, fmaxf(-limx, rx)), cyr = fminf(limy, fmaxf(-limy, ry));
  const float txc = cxr * tz, tyc = cyr * tz;
  const float tz2 = tz * tz, tz3 = tz2 * tz;
  const float j00 = focal_x / tz, j02 = -(focal_x * txc) / tz2, j11 = focal_y / tz, j12 = -(focal_y * tyc) / tz2;
  float R[9];
  quat_to_rot(q, R);
  const float s[3] = {s_in[0] * mod, s_in[1] * mod, s_in[2] * mod};
  float Mq[9];
  for (int i = 0; i < 3; ++i)
    for (int k = 0; k < 3; ++k) Mq[i * 3 + k] = R[i * 3 + k] * s[k];
  float Sg[3][3];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) Sg[i][j] = Mq[i * 3] * Mq[j * 3] + Mq[i * 3 + 1] * Mq[j * 3 + 1] + Mq[i * 3 + 2] * Mq[j * 3 + 2];
  float Rv[3][3];   // Rv[i][k] = vm[4k+i]
  for (int i = 0; i < 3; ++i)
    for (int k = 0; k < 3; ++k) Rv[i][k] = vm[4 * k + i];
  float m0[3], m1[3];
  for (int k = 0; k < 3; ++k) { m0[k] = j00 * Rv[0][k] + j02 * Rv[2][k]; m1[k] = j11 * Rv[1][k] + j12 * Rv[2][k]; }
  float v0[3], v1[3];
  for (int k = 0; k < 3; ++k) {
    v0[k] = Sg[k][0] * m0[0] + Sg[k][1] * m0[1] + Sg[k][2] * m0[2];
    v1[k] = Sg[k][0] * m1[0] + Sg[k][1] * m1[1] + Sg[k][2] * m1[2];
  }
  const float a = m0[0] * v0[0] + m0[1] * v0[1] + m0[2] * v0[2] + 0.3f;
  const float b = m0[0] * v1[0] + m0[1] * v1[1] + m0[2] * v1[2];
  const float c = m1[0] * v1[0] + m1[1] * v1[1] + m1[2] * v1[2] + 0.3f;
  const float det = a * c - b * b;
  const float id2 = 1.0f / (det * det);
  // conic = (c, -b, a) / det
  const float ga = (gA * (-c * c) + gB * (b * c) + gC * (-b * b)) * id2;
  const float gb = (gA * (2.f * b * c) - gB * (det + 2.f * b * b) + gC * (2.f * a * b)) * id2;
  const float gc = (gA * (-b * b) + gB * (a * b) + gC * (-a * a)) * id2;
  // (a,b,c) -> Sigma (full 3x3 gradient, entries treated independently) and m0, m1
  float GS[3][3];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) GS[i][j] = ga * m0[i] * m0[j] + gb * m0[i] * m1[j] + gc * m1[i] * m1[j];
  float gm0[3], gm1[3];
  for (int k = 0; k < 3; ++k) { gm0[k] = 2.f * ga * v0[k] + gb * v1[k]; gm1[k] = 2.f * gc * v1[k] + gb * v0[k]; }
  // M -> J
  float gj00 = 0.f, gj02 = 0.f, gj11 = 0.f, gj12 = 0.f;
  for (int k = 0; k < 3; ++k) {
    gj00 += gm0[k] * Rv[0][k]; gj02 += gm0[k] * Rv[2][k];
    gj11 += gm1[k] * Rv[1][k]; gj12 += gm1[k] * Rv[2][k];
  }
  // J -> t
  const float gtxc = gj02 * (-focal_x / tz2), gtyc = gj12 * (-focal_y / tz2);
  float gtz = gj00 * (-focal_x / tz2) + gj02 * (2.f * focal_x * txc / tz3) + gj11 * (-focal_y / tz2) + gj12 * (2.f * focal_y * tyc / tz3);
  float gtx = 0.f, gty = 0.f;
  if (clx) gtz += gtxc * cxr; else gtx += gtxc;
  if (cly) gtz += gtyc * cyr; else gty += gtyc;
  gtz += gdepth;
  // t -> p
  for (int k = 0; k < 3; ++k) dmean[k] = Rv[0][k] * gtx + Rv[1][k] * gty + Rv[2][k] * gtz;
  // pixel centre -> p
  const float hx = tp(pm, 0), hy = tp(pm, 1), hw = tp(pm, 3);
  const float p_w = 1.0f / (hw + 1e-7f);
  const float gprojx = gpx * 0.5f * (float)W, gprojy = gpy * 0.5f * (float)H;
  const float ghx = gprojx * p_w, ghy = gprojy * p_w;
  const float ghw = -(gprojx * hx + gprojy * hy) * p_w * p_w;
  for (int k = 0; k < 3; ++k) dmean[k] += ghx * pm[4 * k + 0] + ghy * pm[4 * k + 1] + ghw * pm[4 * k + 3];
  // Sigma = Mq Mq^T -> Mq -> (s, R)
  float gM[9];
  for (int i = 0; i < 3; ++i)
    for (int k = 0; k < 3; ++k) {
      float acc = 0.f;
      for (int j = 0; j < 3; ++j) acc += (GS[i][j] + GS[j][i]) * Mq[j * 3 + k];
      gM[i * 3 + k] = acc;
    }
  float gR[9];
  for (int k = 0; k < 3; ++k) {
    float acc = 0.f;
    for (int i = 0; i < 3; ++i) { acc += gM[i * 3 + k] * R[i * 3 + k]; gR[i * 3 + k] = gM[i * 3 + k] * s[k]; }
    dscale[k] = acc * mod;
  }
  const float r = q[0], x = q[1], y = q[2], z = q[3];
  drot[0] = 2.f * (-z * gR[1] + y * gR[2] + z * gR[3] - x * gR[5] - y * gR[6] + x * gR[7]);
  drot[1] = 2.f * (y * gR[1] + z * gR[2] + y * gR[3] - 2.f * x * gR[4] - r * gR[5] + z * gR[6] + r * gR[7] - 2.f * x * gR[8]);
  drot[2] = 2.f * (-2.f * y * gR[0] + x * gR[1] + r * gR[2] + x * gR[3] + z * gR[5] - r * gR[6] + z * gR[7] - 2.f * y * gR[8]);
  drot[3] = 2.f * (-2.f * z * gR[0] - r * gR[1] + x * gR[2] + r * gR[3] - 2.f * z * gR[4] + y * gR[5] + x * gR[6] + y * gR[7]);
}

}  // namespace a3d
