// Rasterizer, per-gaussian stages (compiled with --fmad=false so that the index-defining arithmetic -- radii, tile
// rectangles, depth sort keys -- is bit-identical to oracle/raster_oracle.py): batched-over-cameras preprocess, key
// duplication, tile-range identification, and the per-gaussian backward.  All cameras of a call go through ONE launch of
// each kernel (the reference loops over cameras in Python: gaussian_batch_renderer_4d.py:27).
#include "a3d_raster_ws.cuh"

namespace a3d {

__global__ void raster_preprocess_kernel(RasterDev a, RasterWs ws, int32_t* __restrict__ radii) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= a.num_cams * a.P) return;
  const int cam = idx / a.P, i = idx % a.P;
  const int g = a.per_cam_geometry ? cam : 0;
  const a3d_raster_cam& c = a.cams[cam];
  PreGauss o;
  const size_t gi = (size_t)g * a.P + i;
  const bool ok = preprocess_gaussian(a.means3D + 3 * gi, a.scales + 3 * gi, a.rotations + 4 * gi, a.scale_modifier, c.viewmatrix,
                                      c.projmatrix, c.tanfovx, c.tanfovy, a.H, a.W, o);
  radii[idx] = o.radius;
  ws.tiles[idx] = ok ? (uint32_t)o.tiles : 0u;
  if (!ok) return;
  ws.depth[idx] = o.depth;
  ws.xy[idx] = make_float2(o.px, o.py);
  ws.conic_opac[idx] = make_float4(o.conA, o.conB, o.conC, a.opacities[i]);
  ws.rect[idx] = make_int4(o.rx0, o.ry0, o.rx1, o.ry1);
  float rgb[3];
  uint32_t clamped = 0;
  if (a.colors_precomp) {
    for (int ch = 0; ch < 3; ++ch) rgb[ch] = a.colors_precomp[3 * i + ch];
  } else {
    clamped = sh_colour(a.sh_degree, a.means3D + 3 * gi, c.campos, a.shs + (size_t)i * a.sh_coeffs * 3, rgb);
  }
  ws.rgb_depth[idx] = make_float4(rgb[0], rgb[1], rgb[2], o.depth);
  ws.clamped[idx] = (uint8_t)clamped;
}

__global__ void raster_counts_kernel(RasterWs ws, int P, int cams, long long cap) {
  const int cam = threadIdx.x;
  if (cam < cams) {
    const uint32_t hi = ws.offsets[(size_t)(cam + 1) * P - 1];
    const uint32_t lo = cam ? ws.offsets[(size_t)cam * P - 1] : 0u;
    ws.counters[cam] = (long long)(hi - lo);
  }
  if (cam == 0) {
    const long long total = ws.offsets[(size_t)cams * P - 1];
    ws.counters[cams] = total;
    ws.counters[cams + 1] = total > cap ? 1 : 0;
  }
}

__global__ void raster_duplicate_kernel(RasterDev a, RasterWs ws, int gx, int num_tiles, long long cap) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= a.num_cams * a.P) return;
  if (ws.tiles[idx] == 0) return;
  const int cam = idx / a.P, i = idx % a.P;
  long long off = idx ? ws.offsets[idx - 1] : 0;
  const int4 r = ws.rect[idx];
  const uint32_t dbits = __float_as_uint(ws.depth[idx]);
  for (int y = r.y; y < r.w; ++y)
    for (int x = r.x; x < r.z; ++x) {
      if (off < cap) {
        const uint64_t tile = (uint64_t)cam * num_tiles + (uint64_t)(y * gx + x);
        ws.keys_a[off] = (tile << 31) | dbits;     // depth > 0.2: the sign bit is always 0 and is not sorted (one radix pass less)
        ws.vals_a[off] = (uint32_t)i;
      }
      ++off;
    }
}

__global__ void raster_ranges_kernel(RasterWs ws, long long n, long long total_tiles) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n) return;
  const uint64_t tile = ws.keys_b[idx] >> 31;
  if (tile >= (uint64_t)total_tiles) return;   // padding key
  if (idx == 0 || (ws.keys_b[idx - 1] >> 31) != tile) ws.ranges[tile].x = (uint32_t)idx;
  if (idx == n - 1 || (ws.keys_b[idx + 1] >> 31) != tile) ws.ranges[tile].y = (uint32_t)(idx + 1);
}

// Per-(camera, gaussian) part of the preprocess backward, shared by both kernels, for a visible pair idx (camera cam, geometry
// slot gi): the (dconic, dmean2D, ddepth) gradients pushed through the projection into dm / ds / dr, the dmeans2D write
// (upstream convention: gradient w.r.t. NDC coordinates), and with sh_grad the SH colour backward (sh_backward): dL/drgb
// masked by the forward clamp bits into g, the basis into b, and the view-direction term added to dm.  The colour depends on
// the mean through the view direction even when the SH features themselves are frozen buffers, so sh_grad is set whenever
// colours come from SH and either the SH or the mean gradient is requested.
__device__ __forceinline__ void pair_backward(const RasterDev& a, const RasterWs& ws, int cam, int i, size_t idx, size_t gi, float* dmeans2D,
                                              bool sh_grad, float (&dm)[3], float (&ds)[3], float (&dr)[4], float (&b)[16],
                                              float (&g)[3]) {
  const a3d_raster_cam& c = a.cams[cam];
  const float gpx = ws.g_mean2d[2 * idx], gpy = ws.g_mean2d[2 * idx + 1];
  preprocess_backward(a.means3D + 3 * gi, a.scales + 3 * gi, a.rotations + 4 * gi, a.scale_modifier, c.viewmatrix, c.projmatrix,
                      c.tanfovx, c.tanfovy, a.H, a.W, ws.g_conic[3 * idx], ws.g_conic[3 * idx + 1], ws.g_conic[3 * idx + 2], gpx, gpy,
                      ws.g_depth[idx], dm, ds, dr);
  if (dmeans2D) {
    dmeans2D[3 * idx] = gpx * 0.5f * (float)a.W;
    dmeans2D[3 * idx + 1] = gpy * 0.5f * (float)a.H;
    dmeans2D[3 * idx + 2] = 0.f;
  }
  for (int ch = 0; ch < 3; ++ch) g[ch] = ws.g_rgb[3 * idx + ch];
  if (sh_grad)
    sh_backward(a.sh_degree, a.means3D + 3 * gi, c.campos, a.shs + (size_t)i * a.sh_coeffs * 3, ws.clamped[idx], g, b, dm);
}

// per-gaussian backward: (dconic, dmean2D, ddepth, drgb) of every camera -> means3D / scales / rotations / colors / SH
__global__ void raster_preprocess_backward_kernel(RasterDev a, RasterWs ws, const int32_t* __restrict__ radii,
                                                  float* __restrict__ dmeans3D, float* __restrict__ dscales,
                                                  float* __restrict__ drots, float* __restrict__ dcolors,
                                                  float* __restrict__ dshs, float* __restrict__ dmeans2D) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= a.num_cams * a.P) return;
  if (radii[idx] <= 0) return;
  const int cam = idx / a.P, i = idx % a.P;
  const size_t gi = (size_t)(a.per_cam_geometry ? cam : 0) * a.P + i;
  float dm[3], ds[3], dr[4], b[16], g[3];
  pair_backward(a, ws, cam, i, idx, gi, dmeans2D, !a.colors_precomp && (dshs || dmeans3D), dm, ds, dr, b, g);
  for (int k = 0; k < 3; ++k) {
    if (dmeans3D) atomicAdd(dmeans3D + 3 * gi + k, dm[k]);
    if (dscales) atomicAdd(dscales + 3 * gi + k, ds[k]);
  }
  if (drots) for (int k = 0; k < 4; ++k) atomicAdd(drots + 4 * gi + k, dr[k]);
  if (a.colors_precomp) {
    if (dcolors) for (int ch = 0; ch < 3; ++ch) atomicAdd(dcolors + 3 * i + ch, g[ch]);
  } else if (dshs) {
    const int nb = (a.sh_degree + 1) * (a.sh_degree + 1);
    for (int ch = 0; ch < 3; ++ch) {
      if (g[ch] == 0.f) continue;   // clamped channel (or nothing to add)
#pragma unroll
      for (int k = 0; k < 16; ++k)
        if (k < nb) atomicAdd(dshs + ((size_t)i * a.sh_coeffs + k) * 3 + ch, b[k] * g[ch]);
    }
  }
}

// deterministic backward, stage 1: every (camera, gaussian) sums the records of its pair slots in slot (= tile) order
__global__ void raster_gather_records_kernel(RasterDev a, RasterWs ws, const float* __restrict__ records, float* __restrict__ op_part) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= a.num_cams * a.P) return;
  float acc[10];
#pragma unroll
  for (int k = 0; k < 10; ++k) acc[k] = 0.f;
  if (ws.tiles[idx] != 0) {
    const size_t lo = idx ? ws.offsets[idx - 1] : 0u, hi = ws.offsets[idx];
    for (size_t slot = lo; slot < hi; ++slot) {
      const float2* r = reinterpret_cast<const float2*>(records + slot * 10);
#pragma unroll
      for (int k = 0; k < 5; ++k) {
        const float2 v = r[k];
        acc[2 * k] += v.x; acc[2 * k + 1] += v.y;
      }
    }
  }
  ws.g_mean2d[2 * (size_t)idx] = acc[0]; ws.g_mean2d[2 * (size_t)idx + 1] = acc[1];
  for (int k = 0; k < 3; ++k) ws.g_conic[3 * (size_t)idx + k] = acc[2 + k];
  op_part[idx] = acc[5];
  for (int k = 0; k < 3; ++k) ws.g_rgb[3 * (size_t)idx + k] = acc[6 + k];
  ws.g_depth[idx] = acc[9];
}

// deterministic backward, stage 2: one thread per gaussian walks the cameras in order (same per-camera arithmetic as
// raster_preprocess_backward_kernel) and adds each shared gradient once
__global__ void raster_preprocess_backward_det_kernel(RasterDev a, RasterWs ws, const int32_t* __restrict__ radii,
                                                      const float* __restrict__ op_part, float* __restrict__ dmeans3D,
                                                      float* __restrict__ dscales, float* __restrict__ drots,
                                                      float* __restrict__ dopacity, float* __restrict__ dcolors,
                                                      float* __restrict__ dshs, float* __restrict__ dmeans2D) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= a.P) return;
  float am[3] = {0.f, 0.f, 0.f}, as[3] = {0.f, 0.f, 0.f}, ar[4] = {0.f, 0.f, 0.f, 0.f}, acol[3] = {0.f, 0.f, 0.f}, aop = 0.f;
  float ash[16][3];
#pragma unroll
  for (int k = 0; k < 16; ++k) ash[k][0] = ash[k][1] = ash[k][2] = 0.f;
  const int nb = a.colors_precomp ? 0 : (a.sh_degree + 1) * (a.sh_degree + 1);
  for (int cam = 0; cam < a.num_cams; ++cam) {
    const size_t idx = (size_t)cam * a.P + i;
    aop += op_part[idx];
    if (radii[idx] <= 0) continue;
    const size_t gi = (size_t)(a.per_cam_geometry ? cam : 0) * a.P + i;
    float dm[3], ds[3], dr[4], b[16], g[3];
    pair_backward(a, ws, cam, i, idx, gi, dmeans2D, !a.colors_precomp && (dshs || dmeans3D), dm, ds, dr, b, g);
    if (a.per_cam_geometry) {   // one camera per gradient entry: written directly
      for (int k = 0; k < 3; ++k) {
        if (dmeans3D) dmeans3D[3 * gi + k] += dm[k];
        if (dscales) dscales[3 * gi + k] += ds[k];
      }
      if (drots) for (int k = 0; k < 4; ++k) drots[4 * gi + k] += dr[k];
    } else {
      for (int k = 0; k < 3; ++k) { am[k] += dm[k]; as[k] += ds[k]; }
      for (int k = 0; k < 4; ++k) ar[k] += dr[k];
    }
    if (a.colors_precomp) {
      for (int ch = 0; ch < 3; ++ch) acol[ch] += g[ch];
    } else if (dshs) {
#pragma unroll
      for (int k = 0; k < 16; ++k)
        if (k < nb)
#pragma unroll
          for (int ch = 0; ch < 3; ++ch) ash[k][ch] += b[k] * g[ch];   // g is 0 on clamped channels
    }
  }
  if (dopacity) dopacity[i] += aop;
  if (!a.per_cam_geometry) {
    for (int k = 0; k < 3; ++k) {
      if (dmeans3D) dmeans3D[3 * i + k] += am[k];
      if (dscales) dscales[3 * i + k] += as[k];
    }
    if (drots) for (int k = 0; k < 4; ++k) drots[4 * i + k] += ar[k];
  }
  if (a.colors_precomp) {
    if (dcolors) for (int ch = 0; ch < 3; ++ch) dcolors[3 * i + ch] += acol[ch];
  } else if (dshs) {
#pragma unroll
    for (int k = 0; k < 16; ++k)
      if (k < nb)
        for (int ch = 0; ch < 3; ++ch) dshs[((size_t)i * a.sh_coeffs + k) * 3 + ch] += ash[k][ch];
  }
}

void launch_preprocess(const RasterDev& a, const RasterWs& ws, int32_t* radii, cudaStream_t st) {
  const int n = a.num_cams * a.P;
  raster_preprocess_kernel<<<(n + 255) / 256, 256, 0, st>>>(a, ws, radii);
}
void launch_counts(const RasterWs& ws, int P, int cams, long long cap, cudaStream_t st) {
  raster_counts_kernel<<<1, ((cams + 31) / 32) * 32, 0, st>>>(ws, P, cams, cap);
}
void launch_duplicate(const RasterDev& a, const RasterWs& ws, int gx, int num_tiles, long long cap, cudaStream_t st) {
  const int n = a.num_cams * a.P;
  raster_duplicate_kernel<<<(n + 255) / 256, 256, 0, st>>>(a, ws, gx, num_tiles, cap);
}
void launch_ranges(const RasterWs& ws, long long n, long long total_tiles, cudaStream_t st) {
  raster_ranges_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(ws, n, total_tiles);
}
void launch_preprocess_backward(const RasterDev& a, const RasterWs& ws, const int32_t* radii, float* dmeans3D, float* dscales,
                                float* drots, float* dcolors, float* dshs, float* dmeans2D, cudaStream_t st) {
  const int n = a.num_cams * a.P;
  raster_preprocess_backward_kernel<<<(n + 255) / 256, 256, 0, st>>>(a, ws, radii, dmeans3D, dscales, drots, dcolors, dshs, dmeans2D);
}

void launch_gather_records(const RasterDev& a, const RasterWs& ws, const float* records, float* op_part, cudaStream_t st) {
  const int n = a.num_cams * a.P;
  raster_gather_records_kernel<<<(n + 255) / 256, 256, 0, st>>>(a, ws, records, op_part);
}
void launch_preprocess_backward_det(const RasterDev& a, const RasterWs& ws, const int32_t* radii, const float* op_part, float* dmeans3D,
                                    float* dscales, float* drots, float* dopacity, float* dcolors, float* dshs, float* dmeans2D,
                                    cudaStream_t st) {
  raster_preprocess_backward_det_kernel<<<(a.P + 127) / 128, 128, 0, st>>>(a, ws, radii, op_part, dmeans3D, dscales, drots, dopacity,
                                                                           dcolors, dshs, dmeans2D);
}

}  // namespace a3d
