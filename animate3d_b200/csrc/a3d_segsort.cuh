// Stable grouping of (key, value) pairs by a small integer key, for the deterministic gathers of the deformation and ARAP
// backwards: a CUB radix sort (stable, so values of one key keep their input order) and the [begin, end) range of every key.
#pragma once
#include <cub/cub.cuh>

#include "a3d_carve.h"
#include "a3d_host.cuh"

namespace a3d {

inline int seg_key_bits(uint32_t num_keys) {
  int b = 1;
  while (b < 32 && (1u << b) <= num_keys) ++b;
  return b;
}

inline size_t seg_sort_temp_bytes(int n, uint32_t num_keys) {
  size_t b = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, b, (uint32_t*)nullptr, (uint32_t*)nullptr, (uint32_t*)nullptr, (uint32_t*)nullptr, n, 0,
                                  seg_key_bits(num_keys));
  return b + 256;
}

// keys >= num_keys (invalid entries) sort to the end and get no range
static __global__ void seg_ranges_kernel(const uint32_t* __restrict__ keys, int n, uint32_t num_keys, uint2* __restrict__ ranges) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t k = keys[i];
  if (k >= num_keys) return;
  if (i == 0 || keys[i - 1] != k) ranges[k].x = (uint32_t)i;
  if (i == n - 1 || keys[i + 1] != k) ranges[k].y = (uint32_t)(i + 1);
}

// Sorts (keys_in, vals_in) into (keys_out, vals_out) and fills ranges[num_keys] (empty keys: {0, 0}).
inline int seg_sort(const uint32_t* keys_in, const uint32_t* vals_in, uint32_t* keys_out, uint32_t* vals_out, int n, uint32_t num_keys,
                    uint2* ranges, void* temp, size_t temp_bytes, cudaStream_t st) {
  A3D_CUDA_CHECK(cub::DeviceRadixSort::SortPairs(temp, temp_bytes, keys_in, keys_out, vals_in, vals_out, n, 0, seg_key_bits(num_keys), st));
  A3D_CUDA_CHECK(cudaMemsetAsync(ranges, 0, sizeof(uint2) * num_keys, st));
  seg_ranges_kernel<<<(n + 255) / 256, 256, 0, st>>>(keys_out, n, num_keys, ranges);
  A3D_LAUNCH_CHECK();
  return A3D_OK;
}

}  // namespace a3d
