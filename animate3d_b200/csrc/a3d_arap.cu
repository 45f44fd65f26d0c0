// ARAP regulariser of the 4D-SDS / reconstruction step (SURVEY 8f-3; custom/threestudio-animate3d/systems/util.py:58-117,
// 138-215, called from systems/animate3d.py:215-244): brute-force KNN graph of the control nodes (built once -- the
// gaussians' rest positions are frozen) and one fused kernel for all frames that fits the per-node rotation, evaluates the
// edge energy and scatters its gradient.  The arithmetic lives in a3d_arap_math.h (shared with the CPU harness that checks
// it against the reference's own functions).
#include "a3d_host.cuh"
#include "a3d_arap_math.h"
#include "a3d_segsort.cuh"

namespace a3d {

// K+1 nearest (squared distance ascending, ties by index) of every point among all points; the first one is dropped -- the
// lowest-index point coincident with i, i itself unless a lower-index copy exists (include/a3d.h) --
// pytorch3d.ops.knn_points(points, points, K=K+1)[..., 1:] as the reference uses it (util.py:79-82).
__global__ void __launch_bounds__(128) knn_kernel(const float* __restrict__ pts, int n, int K, int* __restrict__ nbr,
                                                  float* __restrict__ dist2) {
  __shared__ float sp[128 * 3];
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const bool ok = i < n;
  const float px = ok ? pts[3 * i] : 0.f, py = ok ? pts[3 * i + 1] : 0.f, pz = ok ? pts[3 * i + 2] : 0.f;
  float bd[kArapMaxK + 1];
  int bi[kArapMaxK + 1];
  for (int k = 0; k <= K; ++k) { bd[k] = INFINITY; bi[k] = -1; }
  for (int base = 0; base < n; base += 128) {
    const int j = base + threadIdx.x;
    __syncthreads();
    if (j < n) { sp[3 * threadIdx.x] = pts[3 * j]; sp[3 * threadIdx.x + 1] = pts[3 * j + 1]; sp[3 * threadIdx.x + 2] = pts[3 * j + 2]; }
    __syncthreads();
    const int cnt = min(128, n - base);
    if (ok) {
      for (int c = 0; c < cnt; ++c) {
        const float dx = px - sp[3 * c], dy = py - sp[3 * c + 1], dz = pz - sp[3 * c + 2];
        const float d = dx * dx + dy * dy + dz * dz;
        if (d < bd[K]) {                      // strict: an equal distance keeps the earlier index (stable sort order)
          int k = K;
          while (k > 0 && d < bd[k - 1]) { bd[k] = bd[k - 1]; bi[k] = bi[k - 1]; --k; }
          bd[k] = d; bi[k] = base + c;
        }
      }
    }
  }
  if (ok)
    for (int k = 0; k < K; ++k) { nbr[(int64_t)i * K + k] = bi[k + 1]; dist2[(int64_t)i * K + k] = bd[k + 1]; }
}

__global__ void __launch_bounds__(128) arap_kernel(const float* __restrict__ nodes, int Nt, int Nv, const int* __restrict__ nbr, int K,
                                                   const float* __restrict__ weight, const int* __restrict__ sample, int Ns,
                                                   float* __restrict__ err, float* __restrict__ grad) {
  __shared__ float red[4];
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t total = (int64_t)(Nt - 1) * Ns;
  float energy = 0.f;
  if (idx < total) {
    const int t = 1 + (int)(idx / Ns);
    const int si = (int)(idx % Ns);
    const int i = sample ? sample[si] : si;
    if (i >= 0 && i < Nv) {
      float e0[kArapMaxK][3], et[kArapMaxK][3], g0[kArapMaxK][3], gt[kArapMaxK][3], w[kArapMaxK];
      bool valid[kArapMaxK];
      arap_gather(nodes, Nv, nbr, K, weight, i, t, e0, et, w, valid);
      energy = arap_node(K, e0, et, valid, w, gt, g0);
      if (grad) {
        float* gT = grad + (int64_t)t * Nv * 3;
#pragma unroll
        for (int n = 0; n < kArapMaxK; ++n) {
          if (n < K && valid[n]) {
            const int j = nbr[(int64_t)i * K + n];
#pragma unroll
            for (int c = 0; c < 3; ++c) {
              atomicAdd(gT + 3 * (int64_t)i + c, gt[n][c]);
              atomicAdd(gT + 3 * (int64_t)j + c, -gt[n][c]);
              atomicAdd(grad + 3 * (int64_t)i + c, g0[n][c]);
              atomicAdd(grad + 3 * (int64_t)j + c, -g0[n][c]);
            }
          }
        }
      }
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) energy += __shfl_xor_sync(0xffffffffu, energy, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = energy;
  __syncthreads();
  if (threadIdx.x == 0) atomicAdd(err, red[0] + red[1] + red[2] + red[3]);
}

// ---- deterministic variant: records instead of atomics, then fixed-order reductions
// energy [(Nt-1)*Ns]; rec_t / rec_0 [(Nt-1)*Ns][K][3]: the frame-t and frame-0 edge gradients (+ to node i, - to neighbour j)
__global__ void __launch_bounds__(128) arap_records_kernel(const float* __restrict__ nodes, int Nt, int Nv, const int* __restrict__ nbr,
                                                           int K, const float* __restrict__ weight, const int* __restrict__ sample,
                                                           int Ns, float* __restrict__ energy, float* __restrict__ rec_t,
                                                           float* __restrict__ rec_0) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (int64_t)(Nt - 1) * Ns) return;
  const int t = 1 + (int)(idx / Ns);
  const int si = (int)(idx % Ns);
  const int i = sample ? sample[si] : si;
  float e0[kArapMaxK][3], et[kArapMaxK][3], g0[kArapMaxK][3], gt[kArapMaxK][3], w[kArapMaxK];
  bool valid[kArapMaxK];
  float en = 0.f;
  const bool node_ok = i >= 0 && i < Nv;
  if (node_ok) {
    arap_gather(nodes, Nv, nbr, K, weight, i, t, e0, et, w, valid);
    en = arap_node(K, e0, et, valid, w, gt, g0);
  }
  energy[idx] = en;
  for (int n = 0; n < K; ++n)
    for (int c = 0; c < 3; ++c) {
      const bool ok = node_ok && valid[n];
      rec_t[(idx * K + n) * 3 + c] = ok ? gt[n][c] : 0.f;
      rec_0[(idx * K + n) * 3 + c] = ok ? g0[n][c] : 0.f;
    }
}

// one CTA: per-thread strided sums, then a fixed shared-memory tree
__global__ void __launch_bounds__(1024) arap_energy_sum_kernel(const float* __restrict__ energy, int64_t n, float* __restrict__ err) {
  __shared__ float s[1024];
  float a = 0.f;
  for (int64_t k = threadIdx.x; k < n; k += 1024) a += energy[k];
  s[threadIdx.x] = a;
  __syncthreads();
  for (int h = 512; h > 0; h >>= 1) {
    if ((int)threadIdx.x < h) s[threadIdx.x] += s[threadIdx.x + h];
    __syncthreads();
  }
  if (threadIdx.x == 0) *err = s[0];
}

// entry e = (si*K + n)*2 + side of the edge list: side 0 targets node i (+), side 1 its neighbour j (-); invalid -> key Nv
__global__ void arap_targets_kernel(const int* __restrict__ nbr, int K, int Nv, const int* __restrict__ sample, int Ns,
                                    uint32_t* __restrict__ keys, uint32_t* __restrict__ vals) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= 2 * Ns * K) return;
  const int si = e / (2 * K), n = (e >> 1) % K;
  const int i = sample ? sample[si] : si;
  int target = Nv;
  if (i >= 0 && i < Nv) {
    const int j = nbr[(int64_t)i * K + n];
    if (j >= 0 && j < Nv) target = (e & 1) ? j : i;
  }
  keys[e] = (uint32_t)target;
  vals[e] = (uint32_t)e;
}

// grad[t, v] = sum over v's entries in sorted order; frame 0 adds the frame-0 records of frames 1 .. Nt-1 in frame order
__global__ void arap_gather_kernel(const uint2* __restrict__ ranges, const uint32_t* __restrict__ entries, const float* __restrict__ rec_t,
                                   const float* __restrict__ rec_0, int Nt, int Nv, int64_t edges_per_frame, float* __restrict__ grad) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (int64_t)Nt * Nv) return;
  const int t = (int)(idx / Nv), v = (int)(idx % Nv);
  const uint2 r = ranges[v];
  float g[3] = {0.f, 0.f, 0.f};
  const int t_lo = t == 0 ? 1 : t, t_hi = t == 0 ? Nt - 1 : t;
  const float* rec = t == 0 ? rec_0 : rec_t;
  for (int tt = t_lo; tt <= t_hi; ++tt)
    for (uint32_t k = r.x; k < r.y; ++k) {
      const uint32_t e = entries[k];
      // record of (frame tt, sample si, edge n) = (tt-1) * Ns*K + si*K + n, and e >> 1 = si*K + n
      const float* rp = rec + 3 * ((int64_t)(tt - 1) * edges_per_frame + (e >> 1));
      if (e & 1) { g[0] -= rp[0]; g[1] -= rp[1]; g[2] -= rp[2]; }
      else       { g[0] += rp[0]; g[1] += rp[1]; g[2] += rp[2]; }
    }
  grad[3 * idx] = g[0]; grad[3 * idx + 1] = g[1]; grad[3 * idx + 2] = g[2];
}

struct ArapScratch {
  float *energy, *rec_t, *rec_0;
  uint32_t *keys_in, *vals_in, *keys_out, *vals_out;
  uint2* ranges;
  void* temp;
  size_t temp_bytes;
};

static size_t carve_arap(void* base, int Nt, int Nv, int K, int Ns, ArapScratch* s) {
  Carve c{static_cast<char*>(base)};
  const size_t recs = (size_t)(Nt - 1) * Ns, entries = 2 * (size_t)Ns * K;
  ArapScratch w;
  w.energy = c.take<float>(recs);
  w.rec_t = c.take<float>(recs * K * 3);
  w.rec_0 = c.take<float>(recs * K * 3);
  w.keys_in = c.take<uint32_t>(entries);
  w.vals_in = c.take<uint32_t>(entries);
  w.keys_out = c.take<uint32_t>(entries);
  w.vals_out = c.take<uint32_t>(entries);
  w.ranges = c.take<uint2>(Nv);
  w.temp_bytes = seg_sort_temp_bytes((int)entries, (uint32_t)Nv);
  w.temp = c.take<char>(w.temp_bytes);
  if (s) *s = w;
  return c.bytes();
}

}  // namespace a3d

using namespace a3d;

extern "C" int a3d_knn_graph(const float* points, int n, int K, int32_t* nbr, float* dist2, void* stream) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (!points || !nbr || !dist2 || n < 2 || K < 1 || K > kArapMaxK || K >= n)
    return fail(A3D_EINVAL, "a3d_knn_graph: need 1 <= K <= %d < n (got K=%d, n=%d) and non-null buffers", kArapMaxK, K, n);
  knn_kernel<<<(n + 127) / 128, 128, 0, st>>>(points, n, K, nbr, dist2);
  A3D_LAUNCH_CHECK();
  return A3D_OK;
}

extern "C" size_t a3d_arap_scratch_bytes(int Nt, int Nv, int K, int Ns, int deterministic) {
  if (!deterministic || Nt < 1 || Nv < 1 || K < 1 || Ns < 1) return 0;
  return carve_arap(nullptr, Nt, Nv, K, Ns, nullptr);
}

extern "C" int a3d_arap(const float* nodes, int Nt, int Nv, const int32_t* nbr, int K, const float* weight, const int32_t* sample,
                        int Ns, int deterministic, float* err, float* grad, void* scratch, size_t scratch_bytes, void* stream) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (!nodes || !nbr || !err || Nt < 1 || Nv < 1 || K < 1 || K > kArapMaxK)
    return fail(A3D_EINVAL, "a3d_arap: bad arguments (Nt=%d Nv=%d K=%d)", Nt, Nv, K);
  if (!sample) Ns = Nv;
  if (Ns < 1) return fail(A3D_EINVAL, "a3d_arap: empty node sample");
  ArapScratch s;
  if (deterministic) {
    if ((int64_t)Ns * K * 2 > 0x7fffffffll) return fail(A3D_EINVAL, "a3d_arap: too many edges for the deterministic path");
    const size_t need = carve_arap(scratch, Nt, Nv, K, Ns, &s);
    if (!scratch || scratch_bytes < need) return fail(A3D_EINVAL, "a3d_arap: deterministic scratch %zu < %zu bytes", scratch_bytes, need);
  }
  const int64_t total = (int64_t)(Nt - 1) * Ns;
  if (!deterministic || total == 0) {   // the atomic kernel accumulates into err / grad; the fixed-order kernels overwrite them
    A3D_CUDA_CHECK(cudaMemsetAsync(err, 0, sizeof(float), st));
    if (grad) A3D_CUDA_CHECK(cudaMemsetAsync(grad, 0, sizeof(float) * (size_t)Nt * Nv * 3, st));
  }
  if (total == 0) return A3D_OK;
  if (!deterministic) {
    arap_kernel<<<(unsigned)((total + 127) / 128), 128, 0, st>>>(nodes, Nt, Nv, nbr, K, weight, sample, Ns, err, grad);
    A3D_LAUNCH_CHECK();
    return A3D_OK;
  }
  arap_records_kernel<<<(unsigned)((total + 127) / 128), 128, 0, st>>>(nodes, Nt, Nv, nbr, K, weight, sample, Ns, s.energy, s.rec_t,
                                                                      s.rec_0);
  A3D_LAUNCH_CHECK();
  arap_energy_sum_kernel<<<1, 1024, 0, st>>>(s.energy, total, err);
  A3D_LAUNCH_CHECK();
  if (!grad) return A3D_OK;
  const int entries = 2 * Ns * K;
  arap_targets_kernel<<<(entries + 255) / 256, 256, 0, st>>>(nbr, K, Nv, sample, Ns, s.keys_in, s.vals_in);
  A3D_LAUNCH_CHECK();
  if (int r = seg_sort(s.keys_in, s.vals_in, s.keys_out, s.vals_out, entries, (uint32_t)Nv, s.ranges, s.temp, s.temp_bytes, st)) return r;
  const int64_t nodes_total = (int64_t)Nt * Nv;
  arap_gather_kernel<<<(unsigned)((nodes_total + 255) / 256), 256, 0, st>>>(s.ranges, s.vals_out, s.rec_t, s.rec_0, Nt, Nv,
                                                                            (int64_t)Ns * K, grad);
  A3D_LAUNCH_CHECK();
  return A3D_OK;
}
