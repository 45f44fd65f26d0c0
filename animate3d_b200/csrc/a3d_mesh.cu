// Mesh animation support (tools/mesh_animation/mesh2gaussian.py, systems/util.py:300-344): the vertex adjacency of a
// triangle mesh as CSR, the per-vertex statistics mesh2gaussian turns into gaussians, and the per-step random neighbour
// draw of the mesh-edge ARAP graph.  No float atomics and no atomics on any output: every result is bit-identical from run
// to run whatever the launch geometry.
#include <cub/cub.cuh>

#include "a3d_carve.h"
#include "a3d_host.cuh"
#include "a3d_segsort.cuh"

namespace a3d {

constexpr int kMeshMaxK = 12;

// ---- adjacency: 6 directed half-edges per face -> sorted unique (src, dst) keys -> CSR

// key = (src << 32) | dst; a corner index outside [0, V) turns the face's edges into the sentinel src = V (dropped)
__global__ void mesh_half_edges_kernel(const int32_t* __restrict__ faces, int F, int V, uint64_t* __restrict__ keys) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= F) return;
  const int v[3] = {faces[3 * (int64_t)f], faces[3 * (int64_t)f + 1], faces[3 * (int64_t)f + 2]};
  const bool ok = v[0] >= 0 && v[0] < V && v[1] >= 0 && v[1] < V && v[2] >= 0 && v[2] < V;
#pragma unroll
  for (int e = 0; e < 3; ++e) {
    const uint32_t a = (uint32_t)v[e], b = (uint32_t)v[(e + 1) % 3];
    keys[6 * (int64_t)f + 2 * e] = ok ? ((uint64_t)a << 32 | b) : ((uint64_t)V << 32);
    keys[6 * (int64_t)f + 2 * e + 1] = ok ? ((uint64_t)b << 32 | a) : ((uint64_t)V << 32);
  }
}

// 1 for the first occurrence of every valid key of the sorted list
__global__ void mesh_unique_flags_kernel(const uint64_t* __restrict__ keys, int n, int V, int32_t* __restrict__ flags) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  const uint64_t key = keys[k];
  flags[k] = (k == 0 || keys[k - 1] != key) && (key >> 32) < (uint64_t)V;
}

// compacts the unique keys: col[pos] = dst, srcs[pos] = src; the last thread also stores the edge count
__global__ void mesh_compact_kernel(const uint64_t* __restrict__ keys, const int32_t* __restrict__ flags,
                                    const int32_t* __restrict__ pos, int n, int32_t* __restrict__ col, int32_t* __restrict__ srcs,
                                    int64_t* __restrict__ count) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  if (flags[k]) {
    col[pos[k]] = (int32_t)(keys[k] & 0xffffffffu);
    srcs[pos[k]] = (int32_t)(keys[k] >> 32);
  }
  if (k == n - 1) *count = pos[k] + flags[k];
}

// row_ptr[r] = first compacted position whose source is >= r: position p writes the rows (src[p-1], src[p]], and the end
// position E writes the rows after the last source.  Every row is written exactly once.
__global__ void mesh_row_ptr_kernel(const int32_t* __restrict__ srcs, const int64_t* __restrict__ count, int n, int V,
                                    int32_t* __restrict__ row_ptr) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  const int E = (int)*count;
  if (p > E || p > n) return;
  const int lo = p == 0 ? -1 : srcs[p - 1];
  const int hi = p == E ? V : srcs[p];
  for (int r = lo + 1; r <= hi; ++r) row_ptr[r] = p;
}

struct AdjScratch {
  uint64_t *keys_in, *keys_out;
  int32_t *flags, *pos, *srcs;
  int64_t* count;
  void* temp;
  size_t temp_bytes;
};

static int key_end_bit(int V) { return 32 + seg_key_bits((uint32_t)V); }

static size_t carve_adjacency(void* base, int V, int F, AdjScratch* s) {
  Carve c{static_cast<char*>(base)};
  const int n = 6 * F;
  AdjScratch w;
  w.keys_in = c.take<uint64_t>(n);
  w.keys_out = c.take<uint64_t>(n);
  w.flags = c.take<int32_t>(n);
  w.pos = c.take<int32_t>(n);
  w.srcs = c.take<int32_t>(n);
  w.count = c.take<int64_t>(1);
  size_t sort_b = 0, scan_b = 0;
  cub::DeviceRadixSort::SortKeys(nullptr, sort_b, (uint64_t*)nullptr, (uint64_t*)nullptr, n, 0, key_end_bit(V));
  cub::DeviceScan::ExclusiveSum(nullptr, scan_b, (int32_t*)nullptr, (int32_t*)nullptr, n);
  w.temp_bytes = (sort_b > scan_b ? sort_b : scan_b) + 256;
  w.temp = c.take<char>(w.temp_bytes);
  if (s) *s = w;
  return c.bytes();
}

// ---- per-vertex statistics

// mean of |v_j - v_i| per axis over the CSR row of i (CSR order), 0 for an empty row
__global__ void mesh_edge_stats_kernel(const float* __restrict__ verts, int V, const int32_t* __restrict__ row_ptr,
                                       const int32_t* __restrict__ col, float* __restrict__ mean_abs_edge) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= V) return;
  const float x = verts[3 * (int64_t)i], y = verts[3 * (int64_t)i + 1], z = verts[3 * (int64_t)i + 2];
  float s[3] = {0.f, 0.f, 0.f};
  const int b = row_ptr[i], e = row_ptr[i + 1];
  for (int k = b; k < e; ++k) {
    const int64_t j = col[k];
    s[0] += fabsf(verts[3 * j] - x);
    s[1] += fabsf(verts[3 * j + 1] - y);
    s[2] += fabsf(verts[3 * j + 2] - z);
  }
  const float cnt = (float)(e - b);
#pragma unroll
  for (int c = 0; c < 3; ++c) mean_abs_edge[3 * (int64_t)i + c] = e > b ? s[c] / cnt : 0.f;
}

// corner entry c = k * F + f (corner slot k of face f): the reference's three index_add_ passes, one per corner slot
__global__ void mesh_corner_keys_kernel(const int32_t* __restrict__ faces, int F, int V, uint32_t* __restrict__ keys,
                                        uint32_t* __restrict__ vals) {
  const int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= 3 * (int64_t)F) return;
  const int k = (int)(c / F), f = (int)(c % F);
  const int v = faces[3 * (int64_t)f + k];
  keys[c] = (v >= 0 && v < V) ? (uint32_t)v : (uint32_t)V;
  vals[c] = (uint32_t)c;
}

// vertex_rgb[v] = sum of its corners' colours in corner-entry order / max(count, 1)
__global__ void mesh_rgb_kernel(const uint2* __restrict__ ranges, const uint32_t* __restrict__ entries, const float* __restrict__ corner_rgb,
                                int F, int V, float* __restrict__ vertex_rgb) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= V) return;
  const uint2 r = ranges[v];
  float s[3] = {0.f, 0.f, 0.f};
  for (uint32_t q = r.x; q < r.y; ++q) {
    const uint32_t c = entries[q];
    const int64_t k = c / (uint32_t)F, f = c % (uint32_t)F;
    const float* p = corner_rgb + 9 * f + 3 * k;
    s[0] += p[0]; s[1] += p[1]; s[2] += p[2];
  }
  const float cnt = (float)max(r.y - r.x, 1u);
#pragma unroll
  for (int c = 0; c < 3; ++c) vertex_rgb[3 * (int64_t)v + c] = s[c] / cnt;
}

struct StatsScratch {
  uint32_t *keys_in, *vals_in, *keys_out, *vals_out;
  uint2* ranges;
  void* temp;
  size_t temp_bytes;
};

static size_t carve_stats(void* base, int V, int F, StatsScratch* s) {
  Carve c{static_cast<char*>(base)};
  const size_t n = 3 * (size_t)F;
  StatsScratch w;
  w.keys_in = c.take<uint32_t>(n);
  w.vals_in = c.take<uint32_t>(n);
  w.keys_out = c.take<uint32_t>(n);
  w.vals_out = c.take<uint32_t>(n);
  w.ranges = c.take<uint2>(V);
  w.temp_bytes = seg_sort_temp_bytes((int)n, (uint32_t)V);
  w.temp = c.take<char>(w.temp_bytes);
  if (s) *s = w;
  return c.bytes();
}

// ---- neighbour sampling

// Philox4x32-10 (Salmon et al., SC'11): counter (i, j, offset_lo, offset_hi), key (seed_lo, seed_hi); returns word 0
__device__ __forceinline__ uint32_t philox_word0(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint32_t k0, uint32_t k1) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    if (r) { k0 += 0x9E3779B9u; k1 += 0xBB67AE85u; }
    const uint32_t hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
    c0 = hi1 ^ c1 ^ k0; c1 = lo1; c2 = hi0 ^ c3 ^ k1; c3 = lo0;
  }
  return c0;
}

// Per row: every slot j gets the key philox(i, j); the K smallest (key, j) in ascending order are kept in registers
// (insertion with a strict compare, so an equal key keeps the smaller j); missing slots stay -1.  With state non-null,
// (seed, offset) are read from state[0], state[1] instead of the arguments.
__global__ void __launch_bounds__(128) mesh_sample_kernel(const int32_t* __restrict__ row_ptr, const int32_t* __restrict__ col, int V,
                                                          int K, uint64_t seed, uint64_t offset, const uint64_t* __restrict__ state,
                                                          int32_t* __restrict__ nbr) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= V) return;
  if (state) { seed = state[0]; offset = state[1]; }
  uint32_t bk[kMeshMaxK];
  int bj[kMeshMaxK];
#pragma unroll
  for (int k = 0; k < kMeshMaxK; ++k) { bk[k] = 0xffffffffu; bj[k] = -1; }
  const int b = row_ptr[i], deg = row_ptr[i + 1] - b;
  const uint32_t s0 = (uint32_t)seed, s1 = (uint32_t)(seed >> 32), o0 = (uint32_t)offset, o1 = (uint32_t)(offset >> 32);
  int have = 0;
  for (int j = 0; j < deg; ++j) {
    const uint32_t key = philox_word0((uint32_t)i, (uint32_t)j, o0, o1, s0, s1);
    if (have == K && key >= bk[K - 1]) continue;
    if (have < K) ++have;
    // from the top: move larger keys up one slot, then place the new key; unrolled so the arrays stay in registers
    bool placed = false;
#pragma unroll
    for (int q = kMeshMaxK - 1; q >= 0; --q) {
      if (q < have && !placed) {
        if (q > 0 && bk[q - 1] > key) { bk[q] = bk[q - 1]; bj[q] = bj[q - 1]; }
        else { bk[q] = key; bj[q] = j; placed = true; }
      }
    }
  }
#pragma unroll
  for (int k = 0; k < kMeshMaxK; ++k)
    if (k < K) nbr[(int64_t)i * K + k] = bj[k] < 0 ? -1 : col[b + bj[k]];
}

// stream-ordered after the draw that read state[1]
__global__ void mesh_advance_offset_kernel(uint64_t* state) { state[1] += 1; }

}  // namespace a3d

using namespace a3d;

extern "C" size_t a3d_mesh_adjacency_scratch_bytes(int V, int F) {
  if (V < 1 || F < 1 || (int64_t)F * 6 > 0x7fffffffll) return 0;
  return carve_adjacency(nullptr, V, F, nullptr);
}

extern "C" int a3d_mesh_adjacency(const int32_t* faces, int F, int V, int32_t* row_ptr, int32_t* col, int64_t* num_edges_host,
                                  void* scratch, size_t scratch_bytes, void* stream) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (!faces || !row_ptr || !col || !num_edges_host || V < 1 || V >= 0x7fffffff || F < 1 || (int64_t)F * 6 > 0x7fffffffll)
    return fail(A3D_EINVAL, "a3d_mesh_adjacency: bad arguments (F=%d V=%d)", F, V);
  AdjScratch s;
  const size_t need = carve_adjacency(scratch, V, F, &s);
  if (!scratch || scratch_bytes < need) return fail(A3D_EINVAL, "a3d_mesh_adjacency: scratch %zu < %zu bytes", scratch_bytes, need);
  const int n = 6 * F;
  mesh_half_edges_kernel<<<(F + 255) / 256, 256, 0, st>>>(faces, F, V, s.keys_in);
  A3D_LAUNCH_CHECK();
  A3D_CUDA_CHECK(cub::DeviceRadixSort::SortKeys(s.temp, s.temp_bytes, s.keys_in, s.keys_out, n, 0, key_end_bit(V), st));
  mesh_unique_flags_kernel<<<(n + 255) / 256, 256, 0, st>>>(s.keys_out, n, V, s.flags);
  A3D_LAUNCH_CHECK();
  A3D_CUDA_CHECK(cub::DeviceScan::ExclusiveSum(s.temp, s.temp_bytes, s.flags, s.pos, n, st));
  mesh_compact_kernel<<<(n + 255) / 256, 256, 0, st>>>(s.keys_out, s.flags, s.pos, n, col, s.srcs, s.count);
  A3D_LAUNCH_CHECK();
  mesh_row_ptr_kernel<<<(n + 1 + 255) / 256, 256, 0, st>>>(s.srcs, s.count, n, V, row_ptr);
  A3D_LAUNCH_CHECK();
  A3D_CUDA_CHECK(cudaMemcpyAsync(num_edges_host, s.count, sizeof(int64_t), cudaMemcpyDeviceToHost, st));
  return A3D_OK;
}

extern "C" size_t a3d_mesh_vertex_stats_scratch_bytes(int V, int F, int with_rgb) {
  if (!with_rgb || V < 1 || F < 1 || (int64_t)F * 3 > 0x7fffffffll) return 0;
  return carve_stats(nullptr, V, F, nullptr);
}

extern "C" int a3d_mesh_vertex_stats(const float* verts, int V, const int32_t* row_ptr, const int32_t* col, const int32_t* faces, int F,
                                     const float* corner_rgb, float* mean_abs_edge, float* vertex_rgb, void* scratch,
                                     size_t scratch_bytes, void* stream) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (!verts || !row_ptr || !col || !mean_abs_edge || V < 1)
    return fail(A3D_EINVAL, "a3d_mesh_vertex_stats: bad arguments (V=%d)", V);
  mesh_edge_stats_kernel<<<(V + 255) / 256, 256, 0, st>>>(verts, V, row_ptr, col, mean_abs_edge);
  A3D_LAUNCH_CHECK();
  if (!corner_rgb) return A3D_OK;
  if (!faces || !vertex_rgb || F < 1 || (int64_t)F * 3 > 0x7fffffffll)
    return fail(A3D_EINVAL, "a3d_mesh_vertex_stats: colours need faces, vertex_rgb and 1 <= 3F < 2^31 (F=%d)", F);
  StatsScratch s;
  const size_t need = carve_stats(scratch, V, F, &s);
  if (!scratch || scratch_bytes < need) return fail(A3D_EINVAL, "a3d_mesh_vertex_stats: scratch %zu < %zu bytes", scratch_bytes, need);
  const int n = 3 * F;
  mesh_corner_keys_kernel<<<(n + 255) / 256, 256, 0, st>>>(faces, F, V, s.keys_in, s.vals_in);
  A3D_LAUNCH_CHECK();
  if (int r = seg_sort(s.keys_in, s.vals_in, s.keys_out, s.vals_out, n, (uint32_t)V, s.ranges, s.temp, s.temp_bytes, st)) return r;
  mesh_rgb_kernel<<<(V + 255) / 256, 256, 0, st>>>(s.ranges, s.vals_out, corner_rgb, F, V, vertex_rgb);
  A3D_LAUNCH_CHECK();
  return A3D_OK;
}

extern "C" int a3d_mesh_sample_neighbors(const int32_t* row_ptr, const int32_t* col, int V, int K, uint64_t seed, uint64_t offset,
                                         int32_t* nbr, void* stream) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (!row_ptr || !col || !nbr || V < 1 || K < 1 || K > kMeshMaxK)
    return fail(A3D_EINVAL, "a3d_mesh_sample_neighbors: need V >= 1, 1 <= K <= %d (got V=%d, K=%d)", kMeshMaxK, V, K);
  mesh_sample_kernel<<<(V + 127) / 128, 128, 0, st>>>(row_ptr, col, V, K, seed, offset, nullptr, nbr);
  A3D_LAUNCH_CHECK();
  return A3D_OK;
}

extern "C" int a3d_mesh_sample_neighbors_state(const int32_t* row_ptr, const int32_t* col, int V, int K, uint64_t* state, int32_t* nbr,
                                               void* stream) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (!row_ptr || !col || !nbr || !state || V < 1 || K < 1 || K > kMeshMaxK)
    return fail(A3D_EINVAL, "a3d_mesh_sample_neighbors_state: need a state, V >= 1, 1 <= K <= %d (got V=%d, K=%d)", kMeshMaxK, V, K);
  mesh_sample_kernel<<<(V + 127) / 128, 128, 0, st>>>(row_ptr, col, V, K, 0, 0, state, nbr);
  A3D_LAUNCH_CHECK();
  mesh_advance_offset_kernel<<<1, 1, 0, st>>>(state);
  A3D_LAUNCH_CHECK();
  return A3D_OK;
}
