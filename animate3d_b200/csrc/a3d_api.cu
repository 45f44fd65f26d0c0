// liba3d.so -- library-level entry points: init, error string, TMA tensor-map cache.
#include "a3d_host.cuh"

namespace a3d {

static PFN_encodeTiled g_encode = nullptr;
static int g_sms = 0;
static std::mutex g_mu;
static std::unordered_map<MapKey, CUtensorMap*, MapKeyHash> g_maps;

PFN_encodeTiled get_encode_fn() {
  if (g_encode) return g_encode;
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult qres;
  if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres) != cudaSuccess ||
      qres != cudaDriverEntryPointSuccess)
    return nullptr;
  g_encode = reinterpret_cast<PFN_encodeTiled>(fn);
  return g_encode;
}

int sm_count() {
  if (g_sms) return g_sms;
  int dev = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&g_sms, cudaDevAttrMultiProcessorCount, dev);
  return g_sms;
}

int get_tensor_map(const MapKey& key, const CUtensorMap** out) {
  std::lock_guard<std::mutex> lk(g_mu);
  auto it = g_maps.find(key);
  if (it != g_maps.end()) {
    *out = it->second;
    return 0;
  }
  PFN_encodeTiled enc = get_encode_fn();
  if (!enc) return fail(A3D_ECUDA, "cuTensorMapEncodeTiled entry point unavailable");
  cuuint64_t dims[5], strides[4];
  cuuint32_t box[5], estr[5];
  for (int i = 0; i < 5; ++i) {
    dims[i] = key.dims[i];
    box[i] = key.box[i];
    estr[i] = key.estr[i];
  }
  for (int i = 0; i < 4; ++i) strides[i] = key.strides[i] * 2;  // bytes (fp16)
  CUtensorMap* m = new CUtensorMap;
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 5, const_cast<void*>(key.base), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    delete m;
    return fail(A3D_ECUDA,
                "cuTensorMapEncodeTiled failed (%d): base=%p dims=[%llu,%llu,%llu,%llu,%llu] strides(el)=[%llu,%llu,%llu,%llu] "
                "box=[%u,%u,%u,%u,%u] estr=[%u,%u,%u,%u,%u]",
                (int)r, key.base, (unsigned long long)dims[0], (unsigned long long)dims[1], (unsigned long long)dims[2],
                (unsigned long long)dims[3], (unsigned long long)dims[4], (unsigned long long)key.strides[0],
                (unsigned long long)key.strides[1], (unsigned long long)key.strides[2],
                (unsigned long long)key.strides[3], box[0], box[1], box[2], box[3], box[4], estr[0], estr[1], estr[2],
                estr[3], estr[4]);
  }
  g_maps.emplace(key, m);
  *out = m;
  return 0;
}

}  // namespace a3d

extern "C" {

const char* a3d_last_error(void) { return a3d::g_err; }

int a3d_version(void) { return 101; }

int a3d_init(void) {
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return a3d::fail(A3D_ECUDA, "cudaGetDevice: %s", cudaGetErrorString(e));
  int major = 0, minor = 0;
  cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev);
  cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev);
  if (major != 9 || minor != 0) return a3d::fail(A3D_ENOTSUP, "liba3d needs an sm_90 device, found sm_%d%d", major, minor);
  if (!a3d::get_encode_fn()) return a3d::fail(A3D_ECUDA, "cuTensorMapEncodeTiled entry point unavailable");
  a3d::sm_count();
  return A3D_OK;
}

}  // extern "C"
