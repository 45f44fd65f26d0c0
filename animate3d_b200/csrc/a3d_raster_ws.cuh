// Shared declarations of the rasterizer translation units: device argument block, workspace carving, launchers.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/a3d.h"
#include "a3d_carve.h"
#include "a3d_raster_math.h"

namespace a3d {

struct RasterDev {
  int P, H, W, num_cams;
  const a3d_raster_cam* cams;
  const float *means3D, *scales, *rotations, *opacities, *shs, *colors_precomp;
  int sh_degree, sh_coeffs, per_cam_geometry;
  float scale_modifier;
  float bg[3];
};

struct RasterWs {
  // per (camera, gaussian)
  float* depth;
  float2* xy;
  float4* conic_opac;
  float4* rgb_depth;
  int4* rect;
  uint32_t* tiles;
  uint32_t* offsets;
  uint8_t* clamped;
  // binning
  uint64_t *keys_a, *keys_b;
  uint32_t *vals_a, *vals_b;
  uint2* ranges;
  // per pixel (backward state: null in a forward-only workspace)
  uint32_t* n_contrib;
  float* final_T;
  long long* counters;   // [cams] pair counts, [cams] total, [cams+1] overflow flag
  // backward scratch, per (camera, gaussian) (null in a forward-only workspace)
  float *g_mean2d, *g_conic, *g_depth, *g_rgb;
  int32_t* radii;        // forward-only workspace: radii of a caller that asked for none, per (camera, gaussian)
  void* cub_temp;
  size_t cub_bytes;
};

// Carves `base` (may be null for a size query) and returns the bytes needed.  forward_only (the RGBA8 render) leaves out
// the per-pixel backward state and the backward scratch and adds a radii buffer; the training layout is unchanged by it.
inline size_t carve_workspace(void* base, int P, int H, int W, int cams, long long cap, size_t cub_bytes, RasterWs* ws,
                              bool forward_only = false) {
  Carve c{static_cast<char*>(base)};
  const size_t n = (size_t)cams * P;
  const int gx = (W + kTile - 1) / kTile, gy = (H + kTile - 1) / kTile;
  RasterWs w;
  w.depth = c.take<float>(n);
  w.xy = c.take<float2>(n);
  w.conic_opac = c.take<float4>(n);
  w.rgb_depth = c.take<float4>(n);
  w.rect = c.take<int4>(n);
  w.tiles = c.take<uint32_t>(n);
  w.offsets = c.take<uint32_t>(n);
  w.clamped = c.take<uint8_t>(n);
  w.keys_a = c.take<uint64_t>(cap);
  w.keys_b = c.take<uint64_t>(cap);
  w.vals_a = c.take<uint32_t>(cap);
  w.vals_b = c.take<uint32_t>(cap);
  w.ranges = c.take<uint2>((size_t)cams * gx * gy);
  w.n_contrib = nullptr;
  w.final_T = nullptr;
  w.g_mean2d = w.g_conic = w.g_depth = w.g_rgb = nullptr;
  w.radii = nullptr;
  if (forward_only) {
    w.counters = c.take<long long>(cams + 2);
    w.radii = c.take<int32_t>(n);
  } else {
    w.n_contrib = c.take<uint32_t>((size_t)cams * H * W);
    w.final_T = c.take<float>((size_t)cams * H * W);
    w.counters = c.take<long long>(cams + 2);
    w.g_mean2d = c.take<float>(2 * n);
    w.g_conic = c.take<float>(3 * n);
    w.g_depth = c.take<float>(n);
    w.g_rgb = c.take<float>(3 * n);
  }
  w.cub_temp = c.take<char>(cub_bytes);
  w.cub_bytes = cub_bytes;
  if (ws) *ws = w;
  return c.bytes();
}

void launch_preprocess(const RasterDev& a, const RasterWs& ws, int32_t* radii, cudaStream_t st);
void launch_counts(const RasterWs& ws, int P, int cams, long long cap, cudaStream_t st);
void launch_duplicate(const RasterDev& a, const RasterWs& ws, int gx, int num_tiles, long long cap, cudaStream_t st);
void launch_ranges(const RasterWs& ws, long long n, long long total_tiles, cudaStream_t st);
void launch_preprocess_backward(const RasterDev& a, const RasterWs& ws, const int32_t* radii, float* dmeans3D, float* dscales,
                                float* drots, float* dcolors, float* dshs, float* dmeans2D, cudaStream_t st);
// deterministic backward: records [max_rendered][10] -> ws.g_* and op_part [cams, P]; then cameras summed in camera order.
// Slots at or past cap (pairs an overflowing forward dropped) are not read.
void launch_gather_records(const RasterDev& a, const RasterWs& ws, const float* records, float* op_part, long long cap,
                           cudaStream_t st);
void launch_preprocess_backward_det(const RasterDev& a, const RasterWs& ws, const int32_t* radii, const float* op_part, float* dmeans3D,
                                    float* dscales, float* drots, float* dopacity, float* dcolors, float* dshs, float* dmeans2D,
                                    cudaStream_t st);

}  // namespace a3d
