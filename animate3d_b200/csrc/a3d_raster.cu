// Rasterizer: tile-binned splatting, all cameras of a batch in one launch per stage.
//   forward : preprocess -> inclusive scan (CUB) -> duplicate (tile|depth) keys -> radix sort (CUB) -> tile ranges ->
//             one 16x16 CTA per (tile, camera) blending front to back with cooperative shared-memory staging
//   backward: per tile back to front; the per-gaussian partial gradients of the 32 pixels of a warp are reduced with
//             shuffles before ONE atomicAdd per warp (the upstream kernel issues one per pixel), then a per-gaussian kernel
//             pushes (conic, mean2D, depth) gradients through the projection to means3D / scales / rotations
// HBM-bound / ALU-bound integer and fp32 work: no tensor cores here by design.
// Replaces diff_gaussian_rasterization._C.rasterize_gaussians(_backward), called at
// custom/threestudio-animate3d/renderer/diff_gaussian_rasterizer_advanced_4d.py:161-170 of the reference.
#include <cub/cub.cuh>

#include "a3d_host.cuh"
#include "a3d_raster_ws.cuh"

namespace a3d {

constexpr int kBlockPix = kTile * kTile;

// Output mode of the tile render.  kOutFloat: colour / depth / alpha planes plus the backward's n_contrib / final_T.
// kOutRGBA8: one uchar4 per pixel, (clamp01(C + T bg), alpha) quantised as the reference saves its test renders; nothing else.
enum RenderOut { kOutFloat = 0, kOutRGBA8 = 1 };

template <int kOut>
__global__ void __launch_bounds__(kBlockPix)
raster_render_forward_kernel(RasterDev a, RasterWs ws, float* __restrict__ out_color, float* __restrict__ out_depth,
                             float* __restrict__ out_alpha, uchar4* __restrict__ out_rgba) {
  const int gx = (a.W + kTile - 1) / kTile, gy = (a.H + kTile - 1) / kTile;
  const int cam = blockIdx.z;
  const int tile = blockIdx.y * gx + blockIdx.x;
  const int px = blockIdx.x * kTile + threadIdx.x, py = blockIdx.y * kTile + threadIdx.y;
  const bool inside = px < a.W && py < a.H;
  const uint2 range = ws.ranges[(size_t)cam * gx * gy + tile];
  const int rounds = ((int)(range.y - range.x) + kBlockPix - 1) / kBlockPix;
  int todo = (int)(range.y - range.x);
  __shared__ float2 s_xy[kBlockPix];
  __shared__ float4 s_co[kBlockPix];
  __shared__ float4 s_cd[kBlockPix];
  bool done = !inside;
  float T = 1.f, C0 = 0.f, C1 = 0.f, C2 = 0.f, D = 0.f, A = 0.f;
  uint32_t contributor = 0, last = 0;
  const int tid = threadIdx.y * kTile + threadIdx.x;
  const size_t cbase = (size_t)cam * a.P;
  for (int r = 0; r < rounds; ++r, todo -= kBlockPix) {
    if (__syncthreads_count(done) == kBlockPix) break;
    const int progress = r * kBlockPix + tid;
    if (range.x + progress < range.y) {
      const uint32_t id = ws.vals_b[range.x + progress];
      s_xy[tid] = ws.xy[cbase + id];
      s_co[tid] = ws.conic_opac[cbase + id];
      s_cd[tid] = ws.rgb_depth[cbase + id];
    }
    __syncthreads();
    const int n = todo < kBlockPix ? todo : kBlockPix;
    for (int j = 0; !done && j < n; ++j) {
      ++contributor;
      const float4 co = s_co[j];
      const float alpha = splat_alpha(s_xy[j].x, s_xy[j].y, co.x, co.y, co.z, co.w, (float)px, (float)py, nullptr);
      if (alpha == 0.f) continue;
      const float test_T = T * (1.f - alpha);
      if (test_T < 0.0001f) { done = true; continue; }
      const float w = alpha * T;
      const float4 cd = s_cd[j];
      C0 += cd.x * w; C1 += cd.y * w; C2 += cd.z * w; D += cd.w * w; A += w;
      T = test_T;
      last = contributor;
    }
  }
  if (inside && kOut == kOutRGBA8) {
    const size_t hw = (size_t)a.H * a.W, pix = (size_t)py * a.W + px;
    out_rgba[(size_t)cam * hw + pix] = make_uchar4(quantise_u8(clamp01(C0 + T * a.bg[0])), quantise_u8(clamp01(C1 + T * a.bg[1])),
                                                   quantise_u8(clamp01(C2 + T * a.bg[2])), quantise_u8(A));
  } else if (inside) {
    const size_t hw = (size_t)a.H * a.W, pix = (size_t)py * a.W + px;
    out_color[((size_t)cam * 3 + 0) * hw + pix] = C0 + T * a.bg[0];
    out_color[((size_t)cam * 3 + 1) * hw + pix] = C1 + T * a.bg[1];
    out_color[((size_t)cam * 3 + 2) * hw + pix] = C2 + T * a.bg[2];
    out_depth[(size_t)cam * hw + pix] = D;
    out_alpha[(size_t)cam * hw + pix] = A;
    ws.n_contrib[(size_t)cam * hw + pix] = last;
    ws.final_T[(size_t)cam * hw + pix] = T;
  }
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// kDet: instead of atomics, every warp parks its 10 totals of list entry j in s_part[warp][j]; after each round of 256
// entries the CTA adds the 8 warps in warp order and stores one record per (camera, tile, gaussian) pair at the pair's slot
// of the pre-sort (duplicate-kernel) order: offset of (camera, gaussian) + row-major index of the tile in its rect.
constexpr int kRecord = 10;   // dmean2D x, y, dconic a, b, c, dopacity, drgb 0..2, ddepth
constexpr int kWarps = kBlockPix / 32;
constexpr size_t kDetSmem = (size_t)kWarps * kBlockPix * kRecord * sizeof(float);

template <bool kDet>
__global__ void __launch_bounds__(kBlockPix)
raster_render_backward_kernel(RasterDev a, RasterWs ws, const float* __restrict__ dL_dcolor, const float* __restrict__ dL_ddepth,
                              const float* __restrict__ dL_dalpha, float* __restrict__ dL_dopacity, float* __restrict__ records) {
  extern __shared__ float s_part[];   // kDet: [kWarps][kBlockPix][kRecord]
  const int gx = (a.W + kTile - 1) / kTile, gy = (a.H + kTile - 1) / kTile;
  const int cam = blockIdx.z;
  const int tile = blockIdx.y * gx + blockIdx.x;
  const int px = blockIdx.x * kTile + threadIdx.x, py = blockIdx.y * kTile + threadIdx.y;
  const bool inside = px < a.W && py < a.H;
  const uint2 range = ws.ranges[(size_t)cam * gx * gy + tile];
  const int total = (int)(range.y - range.x);
  const int rounds = (total + kBlockPix - 1) / kBlockPix;
  __shared__ uint32_t s_id[kBlockPix];
  __shared__ float2 s_xy[kBlockPix];
  __shared__ float4 s_co[kBlockPix];
  __shared__ float4 s_cd[kBlockPix];
  const size_t hw = (size_t)a.H * a.W, pix = (size_t)py * a.W + px;
  const size_t cbase = (size_t)cam * a.P;
  const float T_final = inside ? ws.final_T[(size_t)cam * hw + pix] : 0.f;
  float T = T_final;
  const int last_contributor = inside ? (int)ws.n_contrib[(size_t)cam * hw + pix] : 0;
  float dC[3] = {0.f, 0.f, 0.f}, dD = 0.f, dA = 0.f;
  if (inside) {
    for (int ch = 0; ch < 3; ++ch) dC[ch] = dL_dcolor[((size_t)cam * 3 + ch) * hw + pix];
    if (dL_ddepth) dD = dL_ddepth[(size_t)cam * hw + pix];
    if (dL_dalpha) dA = dL_dalpha[(size_t)cam * hw + pix];
  }
  float acc_col[3] = {0.f, 0.f, 0.f}, acc_d = 0.f, acc_a = 0.f, last_alpha = 0.f, last_col[3] = {0.f, 0.f, 0.f}, last_d = 0.f;
  const int tid = threadIdx.y * kTile + threadIdx.x;
  const int lane = tid & 31;
  int contributor = total;   // 1-based index (in list order) of the entry about to be processed, counted from the back
  // where lane 2k sends the warp total of value k (see the reduction below); odd lanes and k >= 10 have no target
  float* tgt_base = nullptr;
  size_t tgt_off = cbase;
  int tgt_mul = 1, tgt_add = 0;
  if (!(lane & 1)) {
    switch (lane >> 1) {
      case 0: tgt_base = ws.g_mean2d; tgt_mul = 2; tgt_add = 0; break;
      case 1: tgt_base = ws.g_mean2d; tgt_mul = 2; tgt_add = 1; break;
      case 2: tgt_base = ws.g_conic; tgt_mul = 3; tgt_add = 0; break;
      case 3: tgt_base = ws.g_conic; tgt_mul = 3; tgt_add = 1; break;
      case 4: tgt_base = ws.g_conic; tgt_mul = 3; tgt_add = 2; break;
      case 5: tgt_base = dL_dopacity; tgt_off = 0; break;                 // opacities are shared by the cameras: [P]
      case 6: tgt_base = ws.g_rgb; tgt_mul = 3; tgt_add = 0; break;
      case 7: tgt_base = ws.g_rgb; tgt_mul = 3; tgt_add = 1; break;
      case 8: tgt_base = ws.g_rgb; tgt_mul = 3; tgt_add = 2; break;
      case 9: tgt_base = ws.g_depth; break;
      default: break;
    }
  }
  const int warp_last = __reduce_max_sync(0xffffffffu, last_contributor);   // entries behind every pixel's last one: skip
  for (int r = 0; r < rounds; ++r) {
    __syncthreads();
    const int progress = r * kBlockPix + tid;   // back to front
    if (progress < total) {
      const uint32_t id = ws.vals_b[range.y - 1 - progress];
      s_id[tid] = id;
      s_xy[tid] = ws.xy[cbase + id];
      s_co[tid] = ws.conic_opac[cbase + id];
      s_cd[tid] = ws.rgb_depth[cbase + id];
    }
    __syncthreads();
    const int n = (total - r * kBlockPix) < kBlockPix ? (total - r * kBlockPix) : kBlockPix;
    float* my_part = s_part + (size_t)(tid >> 5) * kBlockPix * kRecord;
    for (int j = 0; j < n; ++j, --contributor) {
      if (contributor > warp_last) {
        if (kDet && lane < kRecord) my_part[j * kRecord + lane] = 0.f;
        continue;
      }
      SplatGrad g;
      g.dmx = g.dmy = g.dconA = g.dconB = g.dconC = g.dopac = g.ddepth = 0.f;
      g.dcol[0] = g.dcol[1] = g.dcol[2] = 0.f;
      bool active = inside && contributor <= last_contributor;
      if (active) {
        const float4 co = s_co[j];
        float G;
        const float alpha = splat_alpha(s_xy[j].x, s_xy[j].y, co.x, co.y, co.z, co.w, (float)px, (float)py, &G);
        if (alpha == 0.f) {
          active = false;
        } else {
          T = T / (1.f - alpha);
          const float4 cd = s_cd[j];
          const float col[3] = {cd.x, cd.y, cd.z};
          splat_backward(s_xy[j].x, s_xy[j].y, co.x, co.y, co.z, co.w, (float)px, (float)py, alpha, G, T, T_final, col, cd.w, dC,
                         dD, dA, a.bg, acc_col, acc_d, acc_a, last_alpha, last_col, last_d, g);
        }
      }
      if (!__any_sync(0xffffffffu, active)) {
        if (kDet && lane < kRecord) my_part[j * kRecord + lane] = 0.f;
        continue;
      }
      // Transposing butterfly: the 10 partial gradients (padded to 16) of the warp's 32 pixels are reduced with 16 shuffles
      // instead of 10 x 5; afterwards lane 2k holds the warp total of value k and lanes 0, 2, ..., 18 issue their ONE atomic
      // in parallel (the upstream kernel: one atomic per pixel and value; round 1 here: 50 shuffles + 10 serial atomics).
      float v[16] = {g.dmx, g.dmy, g.dconA, g.dconB, g.dconC, g.dopac, g.dcol[0], g.dcol[1], g.dcol[2], g.ddepth,
                     0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll
      for (int o = 16, cnt = 8; cnt >= 1; o >>= 1, cnt >>= 1) {
        const bool upper = (lane & o) != 0;
#pragma unroll
        for (int i = 0; i < cnt; ++i) {
          const float send = upper ? v[i] : v[i + cnt];
          const float keep = upper ? v[i + cnt] : v[i];
          v[i] = keep + __shfl_xor_sync(0xffffffffu, send, o);
        }
      }
      const float total = v[0] + __shfl_xor_sync(0xffffffffu, v[0], 1);
      if (kDet) {
        if (!(lane & 1) && lane < 2 * kRecord) my_part[j * kRecord + (lane >> 1)] = total;
      } else if (tgt_base) {
        atomicAdd(tgt_base + tgt_mul * (tgt_off + (size_t)s_id[j]) + tgt_add, total);
      }
    }
    if (kDet) {
      __syncthreads();
      if (tid < n) {
        float rec[kRecord];
#pragma unroll
        for (int k = 0; k < kRecord; ++k) rec[k] = 0.f;
#pragma unroll 1
        for (int w = 0; w < kWarps; ++w)
#pragma unroll
          for (int k = 0; k < kRecord; ++k) rec[k] += s_part[((size_t)w * kBlockPix + tid) * kRecord + k];
        const size_t gi = cbase + s_id[tid];
        const int4 rc = ws.rect[gi];
        const size_t slot = (gi ? ws.offsets[gi - 1] : 0u) + (size_t)(blockIdx.y - rc.y) * (rc.z - rc.x) + (blockIdx.x - rc.x);
        float2* dst = reinterpret_cast<float2*>(records + slot * kRecord);
#pragma unroll
        for (int k = 0; k < kRecord / 2; ++k) dst[k] = make_float2(rec[2 * k], rec[2 * k + 1]);
      }
    }
  }
}

__global__ void raster_keys_export_kernel(const uint64_t* __restrict__ in, uint64_t* __restrict__ out, long long n) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = ((in[i] >> 31) << 32) | (in[i] & 0x7FFFFFFFull);
}

static int sort_bits(long long total_tiles) {
  int b = 0;
  while ((1ll << b) <= total_tiles) ++b;
  return 31 + (b < 1 ? 1 : b);   // key = (global tile << 31) | depth bits without the (always zero) sign bit
}

static size_t cub_temp_bytes(int n_scan, long long cap, int end_bit) {
  size_t b1 = 0, b2 = 0;
  cub::DeviceScan::InclusiveSum(nullptr, b1, (uint32_t*)nullptr, (uint32_t*)nullptr, n_scan);
  cub::DeviceRadixSort::SortPairs(nullptr, b2, (uint64_t*)nullptr, (uint64_t*)nullptr, (uint32_t*)nullptr, (uint32_t*)nullptr,
                                  (int)cap, 0, end_bit);
  return (b1 > b2 ? b1 : b2) + 256;
}

// Launch and workspace layout of a call: tile grid, sort key bits, CUB temp bytes and the carved workspace (base may be null
// for a size query).  The forward, the backward and the binning tap must all agree on it.
struct RasterLayout {
  int gx, gy;
  long long total_tiles;
  int end_bit;
  size_t bytes;
  RasterWs ws;
};

static RasterLayout raster_layout(void* base, int P, int H, int W, int cams, long long cap, bool forward_only = false) {
  RasterLayout l;
  l.gx = (W + kTile - 1) / kTile;
  l.gy = (H + kTile - 1) / kTile;
  l.total_tiles = (long long)cams * l.gx * l.gy;
  l.end_bit = sort_bits(l.total_tiles);
  l.bytes = carve_workspace(base, P, H, W, cams, cap, cub_temp_bytes(cams * P, cap, l.end_bit), &l.ws, forward_only);
  return l;
}

static RasterDev make_dev(const a3d_raster_args* a) {
  RasterDev d;
  d.P = a->P; d.H = a->H; d.W = a->W; d.num_cams = a->num_cams; d.cams = a->cams;
  d.means3D = a->means3D; d.scales = a->scales; d.rotations = a->rotations; d.opacities = a->opacities;
  d.shs = a->shs; d.colors_precomp = a->colors_precomp;
  d.sh_degree = a->sh_degree; d.sh_coeffs = a->sh_coeffs; d.per_cam_geometry = a->per_cam_geometry;
  d.scale_modifier = a->scale_modifier;
  d.bg[0] = a->bg[0]; d.bg[1] = a->bg[1]; d.bg[2] = a->bg[2];
  return d;
}

static int check_args(const a3d_raster_args* a, long long cap) {
  if (!a || a->P <= 0 || a->H <= 0 || a->W <= 0 || a->num_cams <= 0 || a->num_cams > 1024)
    return fail(A3D_EINVAL, "a3d_raster: bad sizes");
  if (!a->cams || !a->means3D || !a->scales || !a->rotations || !a->opacities) return fail(A3D_EINVAL, "a3d_raster: null geometry");
  if (!a->shs && !a->colors_precomp) return fail(A3D_EINVAL, "a3d_raster: need shs or colors_precomp");
  if (a->shs && (a->sh_degree < 0 || a->sh_degree > 3 || a->sh_coeffs < (a->sh_degree + 1) * (a->sh_degree + 1)))
    return fail(A3D_EINVAL, "a3d_raster: bad SH degree/coeffs");
  if (cap <= 0 || cap > 0x7fffffffll) return fail(A3D_EINVAL, "a3d_raster: max_rendered out of range");
  if ((long long)a->num_cams * a->P > 0x7fffffffll) return fail(A3D_EINVAL, "a3d_raster: cams*P too large");
  return 0;
}

// ---- optional per-stage timing (bench.py's splat roofline): CUDA events recorded on the caller's stream at stage boundaries
constexpr int kStages = 8;   // 0 preprocess, 1 scan+counts+duplicate, 2 radix sort, 3 ranges, 4 render fwd, 5 render bwd, 6 preprocess bwd
static bool g_timing = false;
static cudaEvent_t g_ev[kStages + 2];
static bool g_ev_init = false, g_fwd_rec = false, g_bwd_rec = false;
static void stamp(int i, cudaStream_t st) {
  if (g_timing) cudaEventRecord(g_ev[i], st);
}

}  // namespace a3d

using namespace a3d;

extern "C" int a3d_debug_raster_timing(int enable) {
  if (enable && !g_ev_init) {
    for (int i = 0; i < kStages + 2; ++i) A3D_CUDA_CHECK(cudaEventCreate(&g_ev[i]));
    g_ev_init = true;
  }
  g_timing = enable != 0;
  g_fwd_rec = g_bwd_rec = false;
  return A3D_OK;
}

// ms per stage of the LAST forward (0..4) and backward (5, 6) issued with timing enabled; synchronises on the recorded events
extern "C" int a3d_debug_raster_stage_ms(float* out_host8) {
  if (!g_ev_init || !out_host8) return fail(A3D_EINVAL, "a3d_debug_raster_stage_ms: timing was never enabled");
  for (int i = 0; i < kStages; ++i) out_host8[i] = 0.f;
  if (g_fwd_rec) {
    A3D_CUDA_CHECK(cudaEventSynchronize(g_ev[5]));
    for (int i = 0; i < 5; ++i) A3D_CUDA_CHECK(cudaEventElapsedTime(&out_host8[i], g_ev[i], g_ev[i + 1]));
  }
  if (g_bwd_rec) {
    A3D_CUDA_CHECK(cudaEventSynchronize(g_ev[8]));
    for (int i = 5; i < 7; ++i) A3D_CUDA_CHECK(cudaEventElapsedTime(&out_host8[i], g_ev[i + 1], g_ev[i + 2]));
  }
  return A3D_OK;
}

extern "C" size_t a3d_raster_workspace_bytes(int P, int H, int W, int num_cams, int64_t max_rendered) {
  return raster_layout(nullptr, P, H, W, num_cams, max_rendered).bytes;
}

// The carve only adds aligned offsets to its base, so carving over a 256-aligned stand-in address yields the offsets.
extern "C" size_t a3d_raster_counters_offset(int P, int H, int W, int num_cams, int64_t max_rendered) {
  char* const probe = reinterpret_cast<char*>(256);
  const RasterLayout l = raster_layout(probe, P, H, W, num_cams, max_rendered);
  return (size_t)(reinterpret_cast<char*>(l.ws.counters) - probe);
}

// preprocess, scan, key duplication, radix sort and tile ranges: everything of a forward before the tile render
static int forward_binning(const a3d_raster_args* a, const RasterLayout& l, const RasterDev& d, int32_t* radii, int64_t max_rendered,
                           cudaStream_t st) {
  const RasterWs& ws = l.ws;
  const int n = a->num_cams * a->P;
  A3D_CUDA_CHECK(cudaMemsetAsync(ws.keys_a, 0xFF, (size_t)max_rendered * 8, st));
  A3D_CUDA_CHECK(cudaMemsetAsync(ws.ranges, 0, (size_t)l.total_tiles * 8, st));
  stamp(0, st);
  launch_preprocess(d, ws, radii, st);
  A3D_LAUNCH_CHECK();
  stamp(1, st);
  size_t tb = ws.cub_bytes;
  A3D_CUDA_CHECK(cub::DeviceScan::InclusiveSum(ws.cub_temp, tb, ws.tiles, ws.offsets, n, st));
  launch_counts(ws, a->P, a->num_cams, max_rendered, st);
  launch_duplicate(d, ws, l.gx, l.gx * l.gy, max_rendered, st);
  A3D_LAUNCH_CHECK();
  stamp(2, st);
  tb = ws.cub_bytes;
  A3D_CUDA_CHECK(cub::DeviceRadixSort::SortPairs(ws.cub_temp, tb, ws.keys_a, ws.keys_b, ws.vals_a, ws.vals_b, (int)max_rendered, 0,
                                                 l.end_bit, st));
  stamp(3, st);
  launch_ranges(ws, max_rendered, l.total_tiles, st);
  stamp(4, st);
  return A3D_OK;
}

extern "C" int a3d_raster_forward(const a3d_raster_args* a, float* color, float* depth, float* alpha, int32_t* radii,
                                  void* workspace, size_t workspace_bytes, int64_t max_rendered, int64_t* num_rendered_host,
                                  void* stream) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (int r = check_args(a, max_rendered)) return r;
  if (!color || !depth || !alpha || !radii || !workspace) return fail(A3D_EINVAL, "a3d_raster_forward: null output");
  const RasterLayout l = raster_layout(workspace, a->P, a->H, a->W, a->num_cams, max_rendered);
  if (l.bytes > workspace_bytes) return fail(A3D_EINVAL, "a3d_raster_forward: workspace %zu < %zu bytes", workspace_bytes, l.bytes);
  const RasterWs& ws = l.ws;
  const RasterDev d = make_dev(a);
  if (int r = forward_binning(a, l, d, radii, max_rendered, st)) return r;
  dim3 grid(l.gx, l.gy, a->num_cams), block(kTile, kTile);
  raster_render_forward_kernel<kOutFloat><<<grid, block, 0, st>>>(d, ws, color, depth, alpha, nullptr);
  A3D_LAUNCH_CHECK();
  stamp(5, st);
  g_fwd_rec = g_timing;
  if (num_rendered_host)
    A3D_CUDA_CHECK(cudaMemcpyAsync(num_rendered_host, ws.counters, sizeof(long long) * (a->num_cams + 2), cudaMemcpyDeviceToHost, st));
  return A3D_OK;
}

extern "C" size_t a3d_raster_forward_rgba8_workspace_bytes(int P, int H, int W, int num_cams, int64_t max_rendered) {
  return raster_layout(nullptr, P, H, W, num_cams, max_rendered, true).bytes;
}

extern "C" int a3d_raster_forward_rgba8(const a3d_raster_args* a, uint8_t* rgba, int32_t* radii, void* workspace,
                                        size_t workspace_bytes, int64_t max_rendered, int64_t* num_rendered_host, void* stream) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (int r = check_args(a, max_rendered)) return r;
  if (!rgba || !workspace) return fail(A3D_EINVAL, "a3d_raster_forward_rgba8: null output");
  const RasterLayout l = raster_layout(workspace, a->P, a->H, a->W, a->num_cams, max_rendered, true);
  if (l.bytes > workspace_bytes)
    return fail(A3D_EINVAL, "a3d_raster_forward_rgba8: workspace %zu < %zu bytes", workspace_bytes, l.bytes);
  const RasterWs& ws = l.ws;
  const RasterDev d = make_dev(a);
  if (int r = forward_binning(a, l, d, radii ? radii : ws.radii, max_rendered, st)) return r;
  dim3 grid(l.gx, l.gy, a->num_cams), block(kTile, kTile);
  raster_render_forward_kernel<kOutRGBA8><<<grid, block, 0, st>>>(d, ws, nullptr, nullptr, nullptr, reinterpret_cast<uchar4*>(rgba));
  A3D_LAUNCH_CHECK();
  stamp(5, st);
  g_fwd_rec = g_timing;
  if (num_rendered_host)
    A3D_CUDA_CHECK(cudaMemcpyAsync(num_rendered_host, ws.counters, sizeof(long long) * (a->num_cams + 2), cudaMemcpyDeviceToHost, st));
  return A3D_OK;
}

// deterministic backward scratch: one record per pair slot, then the per-(camera, gaussian) opacity partials
static size_t carve_det(void* base, const a3d_raster_args* a, long long cap, float** records, float** op_part) {
  Carve c{static_cast<char*>(base)};
  float* r = c.take<float>((size_t)cap * kRecord);
  float* o = c.take<float>((size_t)a->num_cams * a->P);
  if (records) *records = r;
  if (op_part) *op_part = o;
  return c.bytes();
}

extern "C" size_t a3d_raster_backward_scratch_bytes(const a3d_raster_args* a, int64_t max_rendered) {
  if (!a || !a->deterministic || check_args(a, max_rendered)) return 0;
  return carve_det(nullptr, a, max_rendered, nullptr, nullptr);
}

extern "C" int a3d_raster_backward(const a3d_raster_args* a, const float* dL_dcolor, const float* dL_ddepth, const float* dL_dalpha,
                                   const int32_t* radii, void* workspace, size_t workspace_bytes, int64_t max_rendered,
                                   float* dL_dmeans3D, float* dL_dscales, float* dL_drotations, float* dL_dopacity, float* dL_dcolors,
                                   float* dL_dshs, float* dL_dmeans2D, void* scratch, size_t scratch_bytes, void* stream) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (int r = check_args(a, max_rendered)) return r;
  if (!dL_dcolor || !radii || !workspace) return fail(A3D_EINVAL, "a3d_raster_backward: null input");
  const RasterLayout l = raster_layout(workspace, a->P, a->H, a->W, a->num_cams, max_rendered);
  if (l.bytes > workspace_bytes) return fail(A3D_EINVAL, "a3d_raster_backward: workspace %zu < %zu bytes", workspace_bytes, l.bytes);
  const RasterWs& ws = l.ws;
  float *records = nullptr, *op_part = nullptr;
  if (a->deterministic) {
    const size_t det = carve_det(scratch, a, max_rendered, &records, &op_part);
    if (!scratch || det > scratch_bytes) return fail(A3D_EINVAL, "a3d_raster_backward: deterministic scratch %zu < %zu bytes", scratch_bytes, det);
  }
  const RasterDev d = make_dev(a);
  const size_t n = (size_t)a->num_cams * a->P;
  A3D_CUDA_CHECK(cudaMemsetAsync(ws.g_mean2d, 0, n * 8, st));
  A3D_CUDA_CHECK(cudaMemsetAsync(ws.g_conic, 0, n * 12, st));
  A3D_CUDA_CHECK(cudaMemsetAsync(ws.g_depth, 0, n * 4, st));
  A3D_CUDA_CHECK(cudaMemsetAsync(ws.g_rgb, 0, n * 12, st));
  dim3 grid(l.gx, l.gy, a->num_cams), block(kTile, kTile);
  stamp(6, st);
  if (a->deterministic) {
    static bool attr = false;
    if (!attr) {
      A3D_CUDA_CHECK(cudaFuncSetAttribute(raster_render_backward_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kDetSmem));
      attr = true;
    }
    raster_render_backward_kernel<true><<<grid, block, kDetSmem, st>>>(d, ws, dL_dcolor, dL_ddepth, dL_dalpha, nullptr, records);
  } else {
    raster_render_backward_kernel<false><<<grid, block, 0, st>>>(d, ws, dL_dcolor, dL_ddepth, dL_dalpha, dL_dopacity, nullptr);
  }
  A3D_LAUNCH_CHECK();
  stamp(7, st);
  if (a->deterministic) {
    launch_gather_records(d, ws, records, op_part, max_rendered, st);
    launch_preprocess_backward_det(d, ws, radii, op_part, dL_dmeans3D, dL_dscales, dL_drotations, dL_dopacity, dL_dcolors, dL_dshs,
                                   dL_dmeans2D, st);
  } else {
    launch_preprocess_backward(d, ws, radii, dL_dmeans3D, dL_dscales, dL_drotations, dL_dcolors, dL_dshs, dL_dmeans2D, st);
  }
  A3D_LAUNCH_CHECK();
  stamp(8, st);
  g_bwd_rec = g_timing;
  return A3D_OK;
}

extern "C" int a3d_raster_binning_tap(const void* workspace, int P, int H, int W, int num_cams, int64_t max_rendered, int cam,
                                      uint64_t* keys_out, uint32_t* point_list_out, uint32_t* ranges_out, void* stream) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const RasterLayout l = raster_layout(const_cast<void*>(workspace), P, H, W, num_cams, max_rendered);
  const RasterWs& ws = l.ws;
  // raw copies of the global sorted tables; the host wrapper slices camera `cam` out of them using the counters
  (void)cam;
  if (keys_out) {   // external form of a key: (tile << 32) | depth bits (the upstream rasterizer's layout)
    raster_keys_export_kernel<<<(unsigned)((max_rendered + 255) / 256), 256, 0, st>>>(ws.keys_b, keys_out, max_rendered);
    A3D_LAUNCH_CHECK();
  }
  if (point_list_out) A3D_CUDA_CHECK(cudaMemcpyAsync(point_list_out, ws.vals_b, (size_t)max_rendered * 4, cudaMemcpyDeviceToDevice, st));
  if (ranges_out) A3D_CUDA_CHECK(cudaMemcpyAsync(ranges_out, ws.ranges, (size_t)l.total_tiles * 8, cudaMemcpyDeviceToDevice, st));
  return A3D_OK;
}

extern "C" int a3d_raster_state_tap(const void* workspace, int P, int H, int W, int num_cams, int64_t max_rendered, int cam,
                                    float* xy_out, float* conic_opac_out, float* rgb_depth_out, uint8_t* clamped_out,
                                    uint32_t* n_contrib_out, float* final_T_out, void* stream) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (!workspace || P <= 0 || H <= 0 || W <= 0 || num_cams <= 0 || cam < 0 || cam >= num_cams)
    return fail(A3D_EINVAL, "a3d_raster_state_tap: bad arguments");
  const RasterLayout l = raster_layout(const_cast<void*>(workspace), P, H, W, num_cams, max_rendered);
  const RasterLayout lr = raster_layout(const_cast<void*>(workspace), P, H, W, num_cams, max_rendered, true);
  // the per-(camera, gaussian) records are carved before anything the RGBA8 layout leaves out, so one tap serves both
  if (l.ws.xy != lr.ws.xy || l.ws.conic_opac != lr.ws.conic_opac || l.ws.rgb_depth != lr.ws.rgb_depth || l.ws.clamped != lr.ws.clamped)
    return fail(A3D_EINVAL, "a3d_raster_state_tap: record offsets differ between the forward and RGBA8 workspaces");
  const RasterWs& ws = l.ws;
  const size_t n = (size_t)P, c0 = (size_t)cam * P, hw = (size_t)H * W;
  if (xy_out) A3D_CUDA_CHECK(cudaMemcpyAsync(xy_out, ws.xy + c0, n * sizeof(float2), cudaMemcpyDeviceToDevice, st));
  if (conic_opac_out) A3D_CUDA_CHECK(cudaMemcpyAsync(conic_opac_out, ws.conic_opac + c0, n * sizeof(float4), cudaMemcpyDeviceToDevice, st));
  if (rgb_depth_out) A3D_CUDA_CHECK(cudaMemcpyAsync(rgb_depth_out, ws.rgb_depth + c0, n * sizeof(float4), cudaMemcpyDeviceToDevice, st));
  if (clamped_out) A3D_CUDA_CHECK(cudaMemcpyAsync(clamped_out, ws.clamped + c0, n, cudaMemcpyDeviceToDevice, st));
  if (n_contrib_out)
    A3D_CUDA_CHECK(cudaMemcpyAsync(n_contrib_out, ws.n_contrib + (size_t)cam * hw, hw * 4, cudaMemcpyDeviceToDevice, st));
  if (final_T_out) A3D_CUDA_CHECK(cudaMemcpyAsync(final_T_out, ws.final_T + (size_t)cam * hw, hw * 4, cudaMemcpyDeviceToDevice, st));
  return A3D_OK;
}
