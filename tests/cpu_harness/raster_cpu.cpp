// CPU harness (TEST INFRASTRUCTURE) around animate3d_b200/csrc/a3d_raster_math.h: drives the exact __host__ __device__
// arithmetic the CUDA kernels use through a serial forward/backward so it can be checked against the oracle without a GPU.
// Build: g++ -O1 -ffp-contract=off -shared -fPIC raster_cpu.cpp -o raster_cpu.so   (done by tests/test_raster_cpu.py)
#include <algorithm>
#include <cstring>
#include <vector>

#include "../../animate3d_b200/csrc/a3d_raster_math.h"

using namespace a3d;

// colours of every gaussian: the precomputed rgb [P,3], or with colors == nullptr the SH colour (sh_colour) of shs
// [P, sh_coeffs, 3] at sh_degree seen from campos, with the clamp bits
static std::vector<float> gaussian_colours(int P, const float* means, const float* colors, const float* shs, int sh_degree,
                                           int sh_coeffs, const float* campos, std::vector<uint32_t>& clamped) {
  std::vector<float> col(3 * (size_t)P);
  clamped.assign(P, 0u);
  for (int i = 0; i < P; ++i) {
    if (colors) for (int ch = 0; ch < 3; ++ch) col[3 * i + ch] = colors[3 * i + ch];
    else clamped[i] = sh_colour(sh_degree, means + 3 * i, campos, shs + (size_t)i * sh_coeffs * 3, &col[3 * i]);
  }
  return col;
}

extern "C" {

// colors: precomputed rgb [P,3], or nullptr for SH colours (shs, sh_degree, sh_coeffs, campos).  Optional outputs: the
// records the kernel's render reads (pre_dump [P,8]: depth, px, py, conic a, b, c, tiles, radius; rgb_out [P,3];
// clamped_out [P]) and the RGBA8 bytes of a3d_raster_forward_rgba8 (rgba_out [H,W,4]).  Returns number of (tile, gaussian)
// pairs.
long raster_cpu_forward(int P, const float* means, const float* scales, const float* rots, const float* opac, const float* colors,
                        const float* shs, int sh_degree, int sh_coeffs, const float* campos,
                        const float* vm, const float* pm, float tanfovx, float tanfovy, int H, int W, const float* bg, float mod,
                        float* out_color, float* out_depth, float* out_alpha, int* radii, int* n_contrib, float* final_T,
                        unsigned long long* keys, unsigned int* vals, long cap, long long* ranges, float* pre_dump,
                        float* rgb_out, unsigned char* clamped_out, unsigned char* rgba_out) {
  const int gx = (W + kTile - 1) / kTile, gy = (H + kTile - 1) / kTile;
  std::vector<uint32_t> clamped;
  const std::vector<float> col = gaussian_colours(P, means, colors, shs, sh_degree, sh_coeffs, campos, clamped);
  colors = col.data();
  if (rgb_out) std::memcpy(rgb_out, col.data(), col.size() * sizeof(float));
  if (clamped_out) for (int i = 0; i < P; ++i) clamped_out[i] = (unsigned char)clamped[i];
  std::vector<PreGauss> pre(P);
  std::vector<std::pair<unsigned long long, unsigned int>> kv;
  for (int i = 0; i < P; ++i) {
    preprocess_gaussian(means + 3 * i, scales + 3 * i, rots + 4 * i, mod, vm, pm, tanfovx, tanfovy, H, W, pre[i]);
    radii[i] = pre[i].radius;
    if (pre_dump) {
      float* d = pre_dump + 8 * i;
      d[0] = pre[i].depth; d[1] = pre[i].px; d[2] = pre[i].py; d[3] = pre[i].conA; d[4] = pre[i].conB; d[5] = pre[i].conC;
      d[6] = (float)pre[i].tiles; d[7] = (float)pre[i].radius;
    }
    if (pre[i].tiles == 0) continue;
    unsigned int dbits;
    std::memcpy(&dbits, &pre[i].depth, 4);
    for (int y = pre[i].ry0; y < pre[i].ry1; ++y)
      for (int x = pre[i].rx0; x < pre[i].rx1; ++x)
        kv.push_back({((unsigned long long)(y * gx + x) << 32) | dbits, (unsigned int)i});
  }
  std::stable_sort(kv.begin(), kv.end(), [](auto& a, auto& b) { return a.first < b.first; });
  const long R = (long)kv.size();
  for (long i = 0; i < R && i < cap; ++i) { keys[i] = kv[i].first; vals[i] = kv[i].second; }
  for (int t = 0; t < gx * gy; ++t) ranges[2 * t] = ranges[2 * t + 1] = 0;
  for (long i = 0; i < R; ++i) {
    const long long t = (long long)(kv[i].first >> 32);
    if (i == 0 || (long long)(kv[i - 1].first >> 32) != t) ranges[2 * t] = i;
    if (i == R - 1 || (long long)(kv[i + 1].first >> 32) != t) ranges[2 * t + 1] = i + 1;
  }
  for (int py = 0; py < H; ++py)
    for (int px = 0; px < W; ++px) {
      const int t = (py / kTile) * gx + px / kTile;
      float T = 1.f, C[3] = {0, 0, 0}, D = 0.f, A = 0.f;
      int contributor = 0, last = 0;
      for (long j = ranges[2 * t]; j < ranges[2 * t + 1]; ++j) {
        ++contributor;
        const int id = (int)kv[j].second;
        const PreGauss& g = pre[id];
        const float alpha = splat_alpha(g.px, g.py, g.conA, g.conB, g.conC, opac[id], (float)px, (float)py, nullptr);
        if (alpha == 0.f) continue;
        const float test_T = T * (1.f - alpha);
        if (test_T < 0.0001f) break;
        const float w = alpha * T;
        for (int ch = 0; ch < 3; ++ch) C[ch] += colors[3 * id + ch] * w;
        D += g.depth * w;
        A += w;
        T = test_T;
        last = contributor;
      }
      const long pix = (long)py * W + px;
      for (int ch = 0; ch < 3; ++ch) out_color[(long)ch * H * W + pix] = C[ch] + T * bg[ch];
      out_depth[pix] = D; out_alpha[pix] = A; n_contrib[pix] = last; final_T[pix] = T;
      if (rgba_out) {
        for (int ch = 0; ch < 3; ++ch) rgba_out[4 * pix + ch] = quantise_u8(clamp01(C[ch] + T * bg[ch]));
        rgba_out[4 * pix + 3] = quantise_u8(A);
      }
    }
  return R;
}

// g_colors receives dL/drgb per gaussian; with SH colours g_shs [P, sh_coeffs, 3] receives dL/dsh and g_means also the
// view-direction term of the colour (sh_backward)
void raster_cpu_backward(int P, const float* means, const float* scales, const float* rots, const float* opac, const float* colors,
                         const float* shs, int sh_degree, int sh_coeffs, const float* campos,
                         const float* vm, const float* pm, float tanfovx, float tanfovy, int H, int W, const float* bg, float mod,
                         const unsigned int* vals, const long long* ranges, const int* n_contrib, const float* final_T,
                         const float* dL_dcolor, const float* dL_ddepth, const float* dL_dalpha,
                         float* g_means, float* g_scales, float* g_rots, float* g_opac, float* g_colors, float* g_shs) {
  const int gx = (W + kTile - 1) / kTile;
  std::vector<uint32_t> clamped;
  const bool sh = colors == nullptr;
  const std::vector<float> col = gaussian_colours(P, means, colors, shs, sh_degree, sh_coeffs, campos, clamped);
  colors = col.data();
  std::vector<PreGauss> pre(P);
  for (int i = 0; i < P; ++i) preprocess_gaussian(means + 3 * i, scales + 3 * i, rots + 4 * i, mod, vm, pm, tanfovx, tanfovy, H, W, pre[i]);
  std::vector<float> gcon(3 * (size_t)P, 0.f), gm2(2 * (size_t)P, 0.f), gdep((size_t)P, 0.f);
  for (int py = 0; py < H; ++py)
    for (int px = 0; px < W; ++px) {
      const int t = (py / kTile) * gx + px / kTile;
      const long pix = (long)py * W + px;
      const float Tf = final_T[pix];
      float T = Tf;
      const float dC[3] = {dL_dcolor[pix], dL_dcolor[(long)H * W + pix], dL_dcolor[2L * H * W + pix]};
      const float dD = dL_ddepth ? dL_ddepth[pix] : 0.f, dA = dL_dalpha ? dL_dalpha[pix] : 0.f;
      float acc_col[3] = {0, 0, 0}, acc_d = 0.f, acc_a = 0.f, last_alpha = 0.f, last_col[3] = {0, 0, 0}, last_d = 0.f;
      const long start = ranges[2 * t];
      for (long j = start + n_contrib[pix] - 1; j >= start; --j) {
        const int id = (int)vals[j];
        const PreGauss& g = pre[id];
        float G;
        const float alpha = splat_alpha(g.px, g.py, g.conA, g.conB, g.conC, opac[id], (float)px, (float)py, &G);
        if (alpha == 0.f) continue;
        T = T / (1.f - alpha);
        SplatGrad sg;
        splat_backward(g.px, g.py, g.conA, g.conB, g.conC, opac[id], (float)px, (float)py, alpha, G, T, Tf, colors + 3 * id,
                       g.depth, dC, dD, dA, bg, acc_col, acc_d, acc_a, last_alpha, last_col, last_d, sg);
        gm2[2 * id] += sg.dmx; gm2[2 * id + 1] += sg.dmy;
        gcon[3 * id] += sg.dconA; gcon[3 * id + 1] += sg.dconB; gcon[3 * id + 2] += sg.dconC;
        g_opac[id] += sg.dopac;
        for (int ch = 0; ch < 3; ++ch) g_colors[3 * id + ch] += sg.dcol[ch];
        gdep[id] += sg.ddepth;
      }
    }
  for (int i = 0; i < P; ++i) {
    if (pre[i].tiles == 0) continue;
    float dm[3], ds[3], dr[4];
    preprocess_backward(means + 3 * i, scales + 3 * i, rots + 4 * i, mod, vm, pm, tanfovx, tanfovy, H, W, gcon[3 * i], gcon[3 * i + 1],
                        gcon[3 * i + 2], gm2[2 * i], gm2[2 * i + 1], gdep[i], dm, ds, dr);
    for (int k = 0; k < 3; ++k) { g_means[3 * i + k] += dm[k]; g_scales[3 * i + k] += ds[k]; }
    for (int k = 0; k < 4; ++k) g_rots[4 * i + k] += dr[k];
    if (sh) {
      float g[3] = {g_colors[3 * i], g_colors[3 * i + 1], g_colors[3 * i + 2]}, b[16];
      sh_backward(sh_degree, means + 3 * i, campos, shs + (size_t)i * sh_coeffs * 3, clamped[i], g, b, g_means + 3 * i);
      for (int k = 0; k < (sh_degree + 1) * (sh_degree + 1); ++k)
        for (int ch = 0; ch < 3; ++ch) g_shs[((size_t)i * sh_coeffs + k) * 3 + ch] += b[k] * g[ch];
    }
  }
}
}
