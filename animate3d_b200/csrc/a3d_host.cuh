// Host-side plumbing shared by the .cu files of liba3d.so: error reporting and a cache of rank-5 TMA tensor maps.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdarg.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <mutex>
#include <string>
#include <unordered_map>

#include "../../include/a3d.h"

namespace a3d {

inline thread_local char g_err[512];

inline int fail(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}

// The a3d_*_kernel queries: the kernel name into a caller buffer of n bytes, NUL-terminated; one that does not fit is an error.
inline int kernel_name(char* name, size_t n, const char* fmt, ...) {
  if (!name) return fail(A3D_EINVAL, "kernel name: null buffer");
  va_list ap;
  va_start(ap, fmt);
  const int len = vsnprintf(name, n, fmt, ap);
  va_end(ap);
  if (len < 0 || (size_t)len >= n) return fail(A3D_EINVAL, "kernel name: %zu bytes do not hold the name", n);
  return A3D_OK;
}

#define A3D_CUDA_CHECK(expr)                                                                          \
  do {                                                                                                \
    cudaError_t _e = (expr);                                                                          \
    if (_e != cudaSuccess) return a3d::fail(A3D_ECUDA, "%s:%d %s -> %s", __FILE__, __LINE__, #expr,   \
                                            cudaGetErrorString(_e));                                  \
  } while (0)

#define A3D_LAUNCH_CHECK() A3D_CUDA_CHECK(cudaGetLastError())

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

PFN_encodeTiled get_encode_fn();

// A rank-5 fp16 tensor map with 128B swizzle.  dims/strides in ELEMENTS (stride of dim 0 is 1); box in elements.
struct MapKey {
  const void* base;
  uint64_t dims[5];
  uint64_t strides[4];   // strides of dims 1..4, elements
  uint32_t box[5];
  uint32_t estr[5];
  bool operator==(const MapKey& o) const { return memcmp(this, &o, sizeof(MapKey)) == 0; }
};
struct MapKeyHash {
  size_t operator()(const MapKey& k) const {
    const uint64_t* p = reinterpret_cast<const uint64_t*>(&k);
    size_t h = 1469598103934665603ull;
    for (size_t i = 0; i < sizeof(MapKey) / 8; ++i) h = (h ^ p[i]) * 1099511628211ull;
    return h;
  }
};

// returns 0 on success; *out points into a cache that lives for the process lifetime
int get_tensor_map(const MapKey& key, const CUtensorMap** out);

inline MapKey make_key(const void* base, const uint64_t (&dims)[5], const uint64_t (&strides)[4],
                       const uint32_t (&box)[5]) {
  MapKey k;
  memset(&k, 0, sizeof(k));
  k.base = base;
  for (int i = 0; i < 5; ++i) { k.dims[i] = dims[i]; k.box[i] = box[i]; k.estr[i] = 1; }
  for (int i = 0; i < 4; ++i) k.strides[i] = strides[i];
  return k;
}

int sm_count();

}  // namespace a3d
