// HBM-bound companions of the tensor-core kernels: GroupNorm(+SiLU) on NHWC (incl. the over-frames variant of the motion
// modules), LayerNorm, temporal (F x F) attention, conv_in / conv_out with the reference's layout changes folded in,
// small fp32 linears for the embeddings, nearest upsample, DDIM+CFG update.  All loads/stores are 16-byte vectors on the
// channel-contiguous (token-major) layout.
#include "a3d_common.cuh"
#include "a3d_host.cuh"

namespace a3d {

__device__ __forceinline__ float silu_f(float x) { return x / (1.0f + __expf(-x)); }

__device__ __forceinline__ int64_t perm_row2(int64_t m, int64_t a, int64_t b) {
  if (a == 0) return m;
  const int64_t ab = a * b;
  return (m / ab) * ab + (m % b) * a + (m / b) % a;
}

// ------------------------------------------------------------------------------------------------ GroupNorm
// Both passes: grid (row chunks, samples); a thread owns one 8-channel vector column (fixed for its lifetime, so gamma / beta /
// group statistics are folded into per-thread scale/shift registers once) and walks rows r0 + rsub, + rows_par, ...;
// blockDim = rows_par * (C / 8).  Four independent 16-byte loads in flight per thread.
// rows per block (chunk) is chosen on the host: 128 when that still yields >= ~4 blocks per SM, fewer rows otherwise (the
// over-frames GroupNorm of the motion modules has only B*Nv = 8 samples)

// Statistics are DETERMINISTIC and cancellation-free: no atomics anywhere.  Every thread accumulates its 8 channels around a
// per-channel pivot (the first value it sees), turns them into (n, mean, M2) triples, and triples are merged with Chan's
// parallel-variance formula in a FIXED order: channels -> group slot inside the thread, a shared-memory tree over the
// block's row lanes, a short serial merge over the vectors of a group, one (n, mean, M2) partial per (sample, chunk, group)
// in global memory, and finally one warp per (sample, group) folding the chunk partials (strided, then a shuffle tree).
struct Moments {
  float n, mean, m2;
};

__device__ __forceinline__ Moments merge(const Moments& a, const Moments& b) {
  if (b.n == 0.f) return a;
  if (a.n == 0.f) return b;
  Moments r;
  r.n = a.n + b.n;
  const float d = b.mean - a.mean, w = b.n / r.n;
  r.mean = fmaf(d, w, a.mean);
  r.m2 = a.m2 + b.m2 + d * d * a.n * w;
  return r;
}

__global__ void __launch_bounds__(512)
gn_stats_kernel(const __half* __restrict__ x1, int c1, const __half* __restrict__ x2, int c2, int rows_per_sample, int groups,
                int rows_par, int chunk_rows, float* __restrict__ partials) {
  extern __shared__ float sm[];  // [rows_par][vpr][2 slots][3]
  const int C = c1 + c2;
  const int vpr = C / 8;
  const int cpg = C / groups;
  const int sample = blockIdx.y;
  const int r0 = blockIdx.x * chunk_rows;
  const int r1 = min(r0 + chunk_rows, rows_per_sample);
  const int vec = threadIdx.x % vpr, rsub = threadIdx.x / vpr;
  if (rsub < rows_par) {
    const int c0 = vec * 8;
    const bool first = c0 < c1;
    const int ld = first ? c1 : c2;
    const __half* src = (first ? x1 + c0 : x2 + (c0 - c1)) + (int64_t)sample * rows_per_sample * ld;
    float s[8], q[8], piv[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) { s[i] = 0.f; q[i] = 0.f; piv[i] = 0.f; }
    float cnt = 0.f;
    int r = r0 + rsub;
    if (r < r1) {
      const uint4 v = __ldg(reinterpret_cast<const uint4*>(src + (int64_t)r * ld));
      const __half2* h = reinterpret_cast<const __half2*>(&v);
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float2 f = __half22float2(h[i]);
        piv[2 * i] = f.x; piv[2 * i + 1] = f.y;
      }
    }
    auto add = [&](const uint4& v) {
      const __half2* h = reinterpret_cast<const __half2*>(&v);
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float2 f = __half22float2(h[i]);
        const float a = f.x - piv[2 * i], b = f.y - piv[2 * i + 1];
        s[2 * i] += a; q[2 * i] = fmaf(a, a, q[2 * i]);
        s[2 * i + 1] += b; q[2 * i + 1] = fmaf(b, b, q[2 * i + 1]);
      }
      cnt += 1.f;
    };
    for (; r + 3 * rows_par < r1; r += 4 * rows_par) {
      const uint4 v0 = __ldg(reinterpret_cast<const uint4*>(src + (int64_t)r * ld));
      const uint4 v1 = __ldg(reinterpret_cast<const uint4*>(src + (int64_t)(r + rows_par) * ld));
      const uint4 v2 = __ldg(reinterpret_cast<const uint4*>(src + (int64_t)(r + 2 * rows_par) * ld));
      const uint4 v3 = __ldg(reinterpret_cast<const uint4*>(src + (int64_t)(r + 3 * rows_par) * ld));
      add(v0); add(v1); add(v2); add(v3);
    }
    for (; r < r1; r += rows_par) add(__ldg(reinterpret_cast<const uint4*>(src + (int64_t)r * ld)));
    // the 8 channels of a vector span at most two groups (cpg >= 8): slot 0 = group c0 / cpg, slot 1 = the next one
    const int g0 = c0 / cpg;
    const int split = (g0 + 1) * cpg - c0;
    Moments ma{0.f, 0.f, 0.f}, mb{0.f, 0.f, 0.f};
    if (cnt > 0.f) {
      const float inv = 1.0f / cnt;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        Moments m;
        m.n = cnt;
        m.mean = piv[i] + s[i] * inv;
        m.m2 = fmaxf(q[i] - s[i] * s[i] * inv, 0.f);
        if (i < split) ma = merge(ma, m); else mb = merge(mb, m);
      }
    }
    float* o = sm + ((rsub * vpr + vec) * 2) * 3;
    o[0] = ma.n; o[1] = ma.mean; o[2] = ma.m2;
    o[3] = mb.n; o[4] = mb.mean; o[5] = mb.m2;
  }
  __syncthreads();
  // tree over the row lanes (fixed pairing)
  for (int stride = 1; stride < rows_par; stride *= 2) {
    if (rsub < rows_par && (rsub % (2 * stride)) == 0 && rsub + stride < rows_par) {
      float* a = sm + ((rsub * vpr + vec) * 2) * 3;
      const float* b = sm + (((rsub + stride) * vpr + vec) * 2) * 3;
#pragma unroll
      for (int sl = 0; sl < 2; ++sl) {
        const Moments m = merge(Moments{a[3 * sl], a[3 * sl + 1], a[3 * sl + 2]}, Moments{b[3 * sl], b[3 * sl + 1], b[3 * sl + 2]});
        a[3 * sl] = m.n; a[3 * sl + 1] = m.mean; a[3 * sl + 2] = m.m2;
      }
    }
    __syncthreads();
  }
  // group g: vectors [g*cpg/8, ((g+1)*cpg-1)/8], slot 0 where the vector starts inside g, slot 1 where it started in g-1
  if (threadIdx.x < groups) {
    const int g = threadIdx.x;
    const int v0 = (g * cpg) / 8, v1 = ((g + 1) * cpg - 1) / 8;
    Moments acc{0.f, 0.f, 0.f};
    for (int v = v0; v <= v1; ++v) {
      const int gv = (v * 8) / cpg;                 // group of the vector's first channel
      const float* e = sm + (v * 2 + (gv == g ? 0 : 1)) * 3;
      acc = merge(acc, Moments{e[0], e[1], e[2]});
    }
    float* o = partials + (((int64_t)sample * gridDim.x + blockIdx.x) * groups + g) * 3;
    o[0] = acc.n; o[1] = acc.mean; o[2] = acc.m2;
  }
}

// one warp per (sample, group): fold the chunk partials -> (mean, rstd)
__global__ void gn_finalize_kernel(const float* __restrict__ partials, int chunks, int groups, float eps, float* __restrict__ stats) {
  const int lane = threadIdx.x & 31;
  const int g = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int sample = blockIdx.y;
  if (g >= groups) return;
  Moments acc{0.f, 0.f, 0.f};
  for (int c = lane; c < chunks; c += 32) {
    const float* e = partials + (((int64_t)sample * chunks + c) * groups + g) * 3;
    acc = merge(acc, Moments{e[0], e[1], e[2]});
  }
#pragma unroll
  for (int off = 1; off < 32; off *= 2) {
    Moments o;
    o.n = __shfl_xor_sync(0xffffffffu, acc.n, off);
    o.mean = __shfl_xor_sync(0xffffffffu, acc.mean, off);
    o.m2 = __shfl_xor_sync(0xffffffffu, acc.m2, off);
    // both partners must compute the same value: always merge (lower lane, higher lane)
    acc = (lane & off) ? merge(o, acc) : merge(acc, o);
  }
  if (lane == 0) {
    stats[((int64_t)sample * groups + g) * 2] = acc.mean;
    stats[((int64_t)sample * groups + g) * 2 + 1] = rsqrtf(acc.m2 / acc.n + eps);
  }
}

__global__ void __launch_bounds__(512)
gn_apply_kernel(const __half* __restrict__ x1, int c1, const __half* __restrict__ x2, int c2, const float* __restrict__ gamma,
                const float* __restrict__ beta, __half* __restrict__ y, int rows_per_sample, int groups, float eps, int silu,
                int64_t perm_a, int64_t perm_b, int rows_par, int chunk_rows, const float* __restrict__ stats) {
  (void)eps;
  const int C = c1 + c2;
  const int vpr = C / 8;
  const int cpg = C / groups;
  const int sample = blockIdx.y;
  const int r0 = blockIdx.x * chunk_rows;
  const int r1 = min(r0 + chunk_rows, rows_per_sample);
  const int vec = threadIdx.x % vpr, rsub = threadIdx.x / vpr;
  if (rsub >= rows_par) return;
  const int c0 = vec * 8;
  const bool first = c0 < c1;
  const int ld = first ? c1 : c2;
  const int64_t row_base = (int64_t)sample * rows_per_sample;
  const __half* src = (first ? x1 + c0 : x2 + (c0 - c1)) + row_base * ld;
  // y = x * scale + shift with scale = rstd * gamma, shift = beta - mean * rstd * gamma
  float scale[8], shift[8];
  {
    const int g0 = c0 / cpg, g1 = (c0 + 7) / cpg;
    const int split = (g0 + 1) * cpg - c0;
    const float2 sa = *reinterpret_cast<const float2*>(stats + ((int64_t)sample * groups + g0) * 2);   // (mean, rstd)
    const float2 sb = *reinterpret_cast<const float2*>(stats + ((int64_t)sample * groups + g1) * 2);
    const float mean0 = sa.x, mean1 = sb.x, rstd0 = sa.y, rstd1 = sb.y;
    const float4 ga = __ldg(reinterpret_cast<const float4*>(gamma + c0)), gb = __ldg(reinterpret_cast<const float4*>(gamma + c0) + 1);
    const float4 ba = __ldg(reinterpret_cast<const float4*>(beta + c0)), bb = __ldg(reinterpret_cast<const float4*>(beta + c0) + 1);
    const float gg[8] = {ga.x, ga.y, ga.z, ga.w, gb.x, gb.y, gb.z, gb.w};
    const float be[8] = {ba.x, ba.y, ba.z, ba.w, bb.x, bb.y, bb.z, bb.w};
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const bool second = i >= split;
      scale[i] = (second ? rstd1 : rstd0) * gg[i];
      shift[i] = be[i] - (second ? mean1 : mean0) * scale[i];
    }
  }
  auto emit = [&](const uint4& v, int r) {
    const __half2* h = reinterpret_cast<const __half2*>(&v);
    float t[8];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float2 f = __half22float2(h[i]);
      t[2 * i] = fmaf(f.x, scale[2 * i], shift[2 * i]);
      t[2 * i + 1] = fmaf(f.y, scale[2 * i + 1], shift[2 * i + 1]);
    }
    if (silu) {
#pragma unroll
      for (int i = 0; i < 8; ++i) t[i] = silu_f(t[i]);
    }
    uint4 o;
    uint32_t* ow = reinterpret_cast<uint32_t*>(&o);
#pragma unroll
    for (int i = 0; i < 4; ++i) ow[i] = pack_f16x2(t[2 * i], t[2 * i + 1]);
    const int64_t orow = perm_row2(row_base + r, perm_a, perm_b);
    *reinterpret_cast<uint4*>(y + orow * C + c0) = o;
  };
  int r = r0 + rsub;
  for (; r + 3 * rows_par < r1; r += 4 * rows_par) {
    const uint4 v0 = __ldg(reinterpret_cast<const uint4*>(src + (int64_t)r * ld));
    const uint4 v1 = __ldg(reinterpret_cast<const uint4*>(src + (int64_t)(r + rows_par) * ld));
    const uint4 v2 = __ldg(reinterpret_cast<const uint4*>(src + (int64_t)(r + 2 * rows_par) * ld));
    const uint4 v3 = __ldg(reinterpret_cast<const uint4*>(src + (int64_t)(r + 3 * rows_par) * ld));
    emit(v0, r); emit(v1, r + rows_par); emit(v2, r + 2 * rows_par); emit(v3, r + 3 * rows_par);
  }
  for (; r < r1; r += rows_par) emit(__ldg(reinterpret_cast<const uint4*>(src + (int64_t)r * ld)), r);
}

// ------------------------------------------------------------------------------------------------ GroupNorm backward (d/dx only)
// The VAE encoder sits on the SDS gradient path (animatemv_guidance.py:365-373): y = [silu](xhat * gamma + beta),
// xhat = (x - mean) * rstd.  With g = dL/dy * silu'(.) * gamma:  dL/dx = rstd * (g - mean(g) - xhat * mean(g * xhat)), the means over
// the (rows x C/groups) elements of a (sample, group).  Same thread mapping and the same fixed-order reductions as the forward
// (no atomics): pass 1 -> per (sample, chunk, group) partial sums, a warp per (sample, group) folds them, pass 2 applies.
// mean / rstd come from the forward's statistics buffer.
__device__ __forceinline__ float dsilu_f(float z) {
  const float sg = 1.0f / (1.0f + __expf(-z));
  return sg * (1.0f + z * (1.0f - sg));
}

template <bool kApply>
__global__ void __launch_bounds__(512)
gn_bwd_kernel(const __half* __restrict__ x, const __half* __restrict__ dy, const float* __restrict__ gamma, const float* __restrict__ beta,
              const float* __restrict__ stats, const float* __restrict__ sums, float* __restrict__ partials, __half* __restrict__ dx,
              int C, int rows_per_sample, int groups, int silu, int rows_par, int chunk_rows) {
  extern __shared__ float sm[];  // pass 1: [rows_par][vpr][2 slots][2]
  const int vpr = C / 8;
  const int cpg = C / groups;
  const int sample = blockIdx.y;
  const int r0 = blockIdx.x * chunk_rows;
  const int r1 = min(r0 + chunk_rows, rows_per_sample);
  const int vec = threadIdx.x % vpr, rsub = threadIdx.x / vpr;
  const int c0 = vec * 8;
  const int g0 = c0 / cpg, g1 = (c0 + 7) / cpg;
  const int split = (g0 + 1) * cpg - c0;
  float s1[2] = {0.f, 0.f}, s2[2] = {0.f, 0.f};
  if (rsub < rows_par) {
    const int64_t row_base = (int64_t)sample * rows_per_sample;
    const float2 sa = *reinterpret_cast<const float2*>(stats + ((int64_t)sample * groups + g0) * 2);   // (mean, rstd)
    const float2 sb = *reinterpret_cast<const float2*>(stats + ((int64_t)sample * groups + g1) * 2);
    float ga[8], be[8];
    {
      const float4 a = __ldg(reinterpret_cast<const float4*>(gamma + c0)), b = __ldg(reinterpret_cast<const float4*>(gamma + c0) + 1);
      const float4 c = __ldg(reinterpret_cast<const float4*>(beta + c0)), d = __ldg(reinterpret_cast<const float4*>(beta + c0) + 1);
      ga[0] = a.x; ga[1] = a.y; ga[2] = a.z; ga[3] = a.w; ga[4] = b.x; ga[5] = b.y; ga[6] = b.z; ga[7] = b.w;
      be[0] = c.x; be[1] = c.y; be[2] = c.z; be[3] = c.w; be[4] = d.x; be[5] = d.y; be[6] = d.z; be[7] = d.w;
    }
    float m1[2] = {0.f, 0.f}, m2[2] = {0.f, 0.f};
    if (kApply) {
      const float2 ta = *reinterpret_cast<const float2*>(sums + ((int64_t)sample * groups + g0) * 2);   // (mean g, mean g*xhat)
      const float2 tb = *reinterpret_cast<const float2*>(sums + ((int64_t)sample * groups + g1) * 2);
      m1[0] = ta.x; m2[0] = ta.y; m1[1] = tb.x; m2[1] = tb.y;
    }
    for (int r = r0 + rsub; r < r1; r += rows_par) {
      const uint4 vx = __ldg(reinterpret_cast<const uint4*>(x + (row_base + r) * C + c0));
      const uint4 vd = __ldg(reinterpret_cast<const uint4*>(dy + (row_base + r) * C + c0));
      const __half2* hx = reinterpret_cast<const __half2*>(&vx);
      const __half2* hd = reinterpret_cast<const __half2*>(&vd);
      float out[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const float2 fx = __half22float2(hx[i >> 1]), fd = __half22float2(hd[i >> 1]);
        const float xv = (i & 1) ? fx.y : fx.x, dv = (i & 1) ? fd.y : fd.x;
        const int sl = i >= split ? 1 : 0;
        const float mean = sl ? sb.x : sa.x, rstd = sl ? sb.y : sa.y;
        const float xh = (xv - mean) * rstd;
        float g = dv * ga[i];
        if (silu) g *= dsilu_f(fmaf(xh, ga[i], be[i]));
        if (kApply) {
          out[i] = rstd * (g - m1[sl] - xh * m2[sl]);
        } else {
          s1[sl] += g;
          s2[sl] = fmaf(g, xh, s2[sl]);
        }
      }
      if (kApply) {
        uint4 o;
        uint32_t* ow = reinterpret_cast<uint32_t*>(&o);
#pragma unroll
        for (int i = 0; i < 4; ++i) ow[i] = pack_f16x2(out[2 * i], out[2 * i + 1]);
        *reinterpret_cast<uint4*>(dx + (row_base + r) * C + c0) = o;
      }
    }
  }
  if (kApply) return;
  if (rsub < rows_par) {
    float* o = sm + ((rsub * vpr + vec) * 2) * 2;
    o[0] = s1[0]; o[1] = s2[0]; o[2] = s1[1]; o[3] = s2[1];
  }
  __syncthreads();
  for (int stride = 1; stride < rows_par; stride *= 2) {      // fixed-order tree over the row lanes
    if (rsub < rows_par && (rsub % (2 * stride)) == 0 && rsub + stride < rows_par) {
      float* a = sm + ((rsub * vpr + vec) * 2) * 2;
      const float* b = sm + (((rsub + stride) * vpr + vec) * 2) * 2;
      a[0] += b[0]; a[1] += b[1]; a[2] += b[2]; a[3] += b[3];
    }
    __syncthreads();
  }
  if (threadIdx.x < groups) {
    const int g = threadIdx.x;
    const int v0 = (g * cpg) / 8, v1 = ((g + 1) * cpg - 1) / 8;
    float a1 = 0.f, a2 = 0.f;
    for (int v = v0; v <= v1; ++v) {
      const int gv = (v * 8) / cpg;
      const float* e = sm + (v * 2 + (gv == g ? 0 : 1)) * 2;
      a1 += e[0]; a2 += e[1];
    }
    float* o = partials + (((int64_t)sample * gridDim.x + blockIdx.x) * groups + g) * 2;
    o[0] = a1; o[1] = a2;
  }
}

__global__ void gn_bwd_finalize_kernel(const float* __restrict__ partials, int chunks, int groups, float inv_n, float* __restrict__ sums) {
  const int lane = threadIdx.x & 31;
  const int g = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int sample = blockIdx.y;
  if (g >= groups) return;
  float a1 = 0.f, a2 = 0.f;
  for (int c = lane; c < chunks; c += 32) {
    const float* e = partials + (((int64_t)sample * chunks + c) * groups + g) * 2;
    a1 += e[0]; a2 += e[1];
  }
#pragma unroll
  for (int off = 1; off < 32; off *= 2) {
    a1 += __shfl_xor_sync(0xffffffffu, a1, off);
    a2 += __shfl_xor_sync(0xffffffffu, a2, off);
  }
  if (lane == 0) {
    sums[((int64_t)sample * groups + g) * 2] = a1 * inv_n;
    sums[((int64_t)sample * groups + g) * 2 + 1] = a2 * inv_n;
  }
}

// ------------------------------------------------------------------------------------------------ LayerNorm
// C = 40 * LPR halves per row (320 / 640 / 1280 -> LPR = 8 / 16 / 32 lanes per row, 5 x 16 B per lane, all loads in flight);
// a warp normalises 32 / LPR rows at once, statistics reduced over the LPR lanes with shuffles.
template <int LPR>
__global__ void layer_norm_kernel(const __half* __restrict__ x, const float* __restrict__ gamma,
                                  const float* __restrict__ beta, __half* __restrict__ y, int64_t rows, float eps) {
  constexpr int C = 40 * LPR;
  constexpr int RPW = 32 / LPR;
  const int lane = threadIdx.x & 31;
  const int64_t row = ((int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5)) * RPW + lane / LPR;
  const int sub = lane % LPR;
  const bool ok = row < rows;
  float v[40];
  float s = 0.f;
  if (ok) {
    const uint4* src = reinterpret_cast<const uint4*>(x + row * C);
    uint4 u[5];
#pragma unroll
    for (int it = 0; it < 5; ++it) u[it] = __ldg(src + sub + it * LPR);
#pragma unroll
    for (int it = 0; it < 5; ++it) {
      const __half2* h = reinterpret_cast<const __half2*>(&u[it]);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 f = __half22float2(h[j]);
        v[it * 8 + 2 * j] = f.x; v[it * 8 + 2 * j + 1] = f.y;
        s += f.x + f.y;
      }
    }
  }
#pragma unroll
  for (int o = LPR / 2; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  const float mean = s / (float)C;
  float q = 0.f;
  if (ok) {
#pragma unroll
    for (int j = 0; j < 40; ++j) { const float d = v[j] - mean; q += d * d; }
  }
#pragma unroll
  for (int o = LPR / 2; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
  const float rstd = rsqrtf(q / (float)C + eps);
  if (ok) {
    uint4* dst = reinterpret_cast<uint4*>(y + row * C);
#pragma unroll
    for (int it = 0; it < 5; ++it) {
      const int c = (sub + it * LPR) * 8;
      const float4 g0 = __ldg(reinterpret_cast<const float4*>(gamma + c)), g1 = __ldg(reinterpret_cast<const float4*>(gamma + c) + 1);
      const float4 b0 = __ldg(reinterpret_cast<const float4*>(beta + c)), b1 = __ldg(reinterpret_cast<const float4*>(beta + c) + 1);
      const float gg[8] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w};
      const float bb[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
      uint4 o;
      uint32_t* ow = reinterpret_cast<uint32_t*>(&o);
#pragma unroll
      for (int j = 0; j < 4; ++j)
        ow[j] = pack_f16x2((v[it * 8 + 2 * j] - mean) * rstd * gg[2 * j] + bb[2 * j],
                           (v[it * 8 + 2 * j + 1] - mean) * rstd * gg[2 * j + 1] + bb[2 * j + 1]);
      dst[sub + it * LPR] = o;
    }
  }
}

// generic fallback (any C % 8 == 0, C <= 1280): one warp per row
__global__ void layer_norm_generic_kernel(const __half* __restrict__ x, const float* __restrict__ gamma,
                                          const float* __restrict__ beta, __half* __restrict__ y, int64_t rows, int C, float eps) {
  const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int lane = threadIdx.x & 31;
  float s = 0.f, q = 0.f;
  for (int c = lane; c < C; c += 32) s += __half2float(x[row * C + c]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  const float mean = s / (float)C;
  for (int c = lane; c < C; c += 32) { const float d = __half2float(x[row * C + c]) - mean; q += d * d; }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
  const float rstd = rsqrtf(q / (float)C + eps);
  for (int c = lane; c < C; c += 32)
    y[row * C + c] = __float2half_rn((__half2float(x[row * C + c]) - mean) * rstd * gamma[c] + beta[c]);
}

// ------------------------------------------------------------------------------------------------ temporal attention
// one block per pixel; thread = (head, query frame).  K/V rows of the pixel are staged in shared memory (all queries of
// a head read the same K/V address -> broadcast); the thread's query row lives in registers.
template <int D>
__global__ void temporal_attn_kernel(const __half* __restrict__ qkv, __half* __restrict__ out, int frames, int heads, float scale,
                                     int64_t ldo) {
  extern __shared__ __align__(16) uint8_t smraw[];
  __half* s = reinterpret_cast<__half*>(smraw);          // [frames][2*C]: k | v
  const int C = heads * D;
  const int64_t pix = blockIdx.x;
  const __half* base = qkv + pix * frames * 3 * C;
  const int vec_row = 2 * C / 8;
  for (int i = threadIdx.x; i < frames * vec_row; i += blockDim.x) {
    const int f = i / vec_row, v = i % vec_row;
    reinterpret_cast<uint4*>(s)[i] = __ldg(reinterpret_cast<const uint4*>(base + (int64_t)f * 3 * C + C) + v);
  }
  const int f = threadIdx.x % frames;
  const int h = threadIdx.x / frames;
  uint4 qreg[D / 8];
  if (h < heads) {
#pragma unroll
    for (int c = 0; c < D / 8; ++c) qreg[c] = __ldg(reinterpret_cast<const uint4*>(base + (int64_t)f * 3 * C + h * D) + c);
  }
  __syncthreads();
  if (h >= heads) return;
  float sc[32];
  float mx = -INFINITY;
  for (int j = 0; j < frames; ++j) {
    const uint4* k = reinterpret_cast<const uint4*>(s + j * 2 * C + h * D);
    float acc = 0.f;
#pragma unroll
    for (int c = 0; c < D / 8; ++c) {
      const uint4 ka = k[c];
      const __half2* qh = reinterpret_cast<const __half2*>(&qreg[c]);
      const __half2* kh = reinterpret_cast<const __half2*>(&ka);
#pragma unroll
      for (int t = 0; t < 4; ++t) {
        const float2 a = __half22float2(qh[t]), b = __half22float2(kh[t]);
        acc = fmaf(a.x, b.x, acc);
        acc = fmaf(a.y, b.y, acc);
      }
    }
    sc[j] = acc * scale;
    mx = fmaxf(mx, sc[j]);
  }
  float sum = 0.f;
  for (int j = 0; j < frames; ++j) { sc[j] = __expf(sc[j] - mx); sum += sc[j]; }
  const float inv = 1.0f / sum;
  __half* o = out + (pix * frames + f) * ldo + h * D;
#pragma unroll
  for (int c = 0; c < D / 8; ++c) {
    float acc[8];
#pragma unroll
    for (int t = 0; t < 8; ++t) acc[t] = 0.f;
    for (int j = 0; j < frames; ++j) {
      const uint4 va = *reinterpret_cast<const uint4*>(s + j * 2 * C + C + h * D + c * 8);
      const __half2* vh = reinterpret_cast<const __half2*>(&va);
#pragma unroll
      for (int t = 0; t < 4; ++t) {
        const float2 b = __half22float2(vh[t]);
        acc[2 * t] = fmaf(sc[j], b.x, acc[2 * t]);
        acc[2 * t + 1] = fmaf(sc[j], b.y, acc[2 * t + 1]);
      }
    }
    uint4 ov;
    uint32_t* ow = reinterpret_cast<uint32_t*>(&ov);
#pragma unroll
    for (int t = 0; t < 4; ++t) ow[t] = pack_f16x2(acc[2 * t] * inv, acc[2 * t + 1] * inv);
    *reinterpret_cast<uint4*>(o + c * 8) = ov;
  }
}

// F == 16 (the shipped motion modules): one block per pixel, one warp per head, the whole 16 x 16 attention of a head as
// mma.sync.m16n8k16 tiles (a 16-frame problem is far below a 64-row wgmma tile; the warp-level MMA is the right size).
// The pixel's [16 frames, 3C] slab is staged in shared memory with coalesced 16-byte loads (rows padded by 16 B so the
// fragment loads of the 8 row groups hit different banks); S and P never leave registers (the accumulator fragment of QK^T
// is exactly the A fragment of P V); the normalised O goes back over the head's dead Q slice and leaves with coalesced
// 16-byte stores.  ~100 warp instructions per (pixel, head) instead of ~1500 in the scalar kernel: HBM-bound.

// HB heads per block (grid.y = heads / HB): 8 x 40, 4 x 80, 2 x 160 channels -> every block stages 16 x 960 halves (31 KB), so
// the wide levels keep ~7 blocks per SM instead of one 123 KB block.
template <int D, int HB>
__global__ void __launch_bounds__(HB * 32) temporal_attn16_kernel(const __half* __restrict__ qkv, __half* __restrict__ out, int heads,
                                                                 float scale_log2, int64_t ldo) {
  extern __shared__ __align__(16) uint8_t smraw[];
  const int C = heads * D;
  constexpr int CB = HB * D;                   // channels of this block's heads
  constexpr int ld = 3 * CB + 8;               // padded row (halves): [q | k | v] of the block's heads
  __half* sm = reinterpret_cast<__half*>(smraw);
  const int64_t pix = blockIdx.x;
  const int hb0 = blockIdx.y * HB;
  const __half* base = qkv + pix * 16 * 3 * C + hb0 * D;
  constexpr int vseg = CB / 8;                 // 16-byte vectors per (row, q|k|v) segment
  for (int i = threadIdx.x; i < 16 * 3 * vseg; i += blockDim.x) {
    const int f = i / (3 * vseg), rem = i % (3 * vseg), part = rem / vseg, v = rem % vseg;
    *reinterpret_cast<uint4*>(sm + f * ld + part * CB + v * 8) =
        __ldg(reinterpret_cast<const uint4*>(base + (int64_t)f * 3 * C + (int64_t)part * C) + v);
  }
  __syncthreads();
  const int h = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;
  {
    const __half* q = sm + h * D;
    const __half* k = sm + CB + h * D;
    const __half* v = sm + 2 * CB + h * D;
    // ---- S = Q K^T: two 8-key n-tiles, ceil(D / 16) k-steps (the last one half empty when D % 16 == 8)
    float s0[4] = {0.f, 0.f, 0.f, 0.f}, s1[4] = {0.f, 0.f, 0.f, 0.f};
    constexpr int KS = (D + 15) / 16;
#pragma unroll
    for (int kk = 0; kk < KS; ++kk) {
      const int d0 = kk * 16 + 2 * t;
      const bool hi_ok = (kk * 16 + 8) < D;    // second 8-column half of this k-step inside the head?
      uint32_t a[4];
      a[0] = *reinterpret_cast<const uint32_t*>(q + g * ld + d0);
      a[1] = *reinterpret_cast<const uint32_t*>(q + (g + 8) * ld + d0);
      a[2] = hi_ok ? *reinterpret_cast<const uint32_t*>(q + g * ld + d0 + 8) : 0u;
      a[3] = hi_ok ? *reinterpret_cast<const uint32_t*>(q + (g + 8) * ld + d0 + 8) : 0u;
      const uint32_t b00 = *reinterpret_cast<const uint32_t*>(k + g * ld + d0);
      const uint32_t b01 = hi_ok ? *reinterpret_cast<const uint32_t*>(k + g * ld + d0 + 8) : 0u;
      const uint32_t b10 = *reinterpret_cast<const uint32_t*>(k + (g + 8) * ld + d0);
      const uint32_t b11 = hi_ok ? *reinterpret_cast<const uint32_t*>(k + (g + 8) * ld + d0 + 8) : 0u;
      mma_16816(s0, a, b00, b01);
      mma_16816(s1, a, b10, b11);
    }
    // ---- softmax over the 16 keys of rows g (c0,c1) and g+8 (c2,c3); a row lives in the 4 lanes of a quad
    float mx_lo = fmaxf(fmaxf(s0[0], s0[1]), fmaxf(s1[0], s1[1]));
    float mx_hi = fmaxf(fmaxf(s0[2], s0[3]), fmaxf(s1[2], s1[3]));
#pragma unroll
    for (int o = 1; o <= 2; o <<= 1) {
      mx_lo = fmaxf(mx_lo, __shfl_xor_sync(0xffffffffu, mx_lo, o));
      mx_hi = fmaxf(mx_hi, __shfl_xor_sync(0xffffffffu, mx_hi, o));
    }
    const float nl = -mx_lo * scale_log2, nh = -mx_hi * scale_log2;
    float p0[4], p1[4];
    p0[0] = ex2_approx(fmaf(s0[0], scale_log2, nl)); p0[1] = ex2_approx(fmaf(s0[1], scale_log2, nl));
    p0[2] = ex2_approx(fmaf(s0[2], scale_log2, nh)); p0[3] = ex2_approx(fmaf(s0[3], scale_log2, nh));
    p1[0] = ex2_approx(fmaf(s1[0], scale_log2, nl)); p1[1] = ex2_approx(fmaf(s1[1], scale_log2, nl));
    p1[2] = ex2_approx(fmaf(s1[2], scale_log2, nh)); p1[3] = ex2_approx(fmaf(s1[3], scale_log2, nh));
    float sum_lo = p0[0] + p0[1] + p1[0] + p1[1], sum_hi = p0[2] + p0[3] + p1[2] + p1[3];
#pragma unroll
    for (int o = 1; o <= 2; o <<= 1) {
      sum_lo += __shfl_xor_sync(0xffffffffu, sum_lo, o);
      sum_hi += __shfl_xor_sync(0xffffffffu, sum_hi, o);
    }
    const float inv_lo = 1.0f / sum_lo, inv_hi = 1.0f / sum_hi;
    // P as the A fragment of the PV product (normalised first: fp16 P in [0,1])
    uint32_t pa[4];
    pa[0] = pack_f16x2(p0[0] * inv_lo, p0[1] * inv_lo);
    pa[1] = pack_f16x2(p0[2] * inv_hi, p0[3] * inv_hi);
    pa[2] = pack_f16x2(p1[0] * inv_lo, p1[1] * inv_lo);
    pa[3] = pack_f16x2(p1[2] * inv_hi, p1[3] * inv_hi);
    // ---- O = P V, 8 value columns per n-tile; V^T fragments through ldmatrix.trans (rows = key frames)
    __syncwarp();
    __half* orow_lo = sm + g * ld + h * D;          // the head's Q slice is dead now: O overwrites it
    __half* orow_hi = sm + (g + 8) * ld + h * D;
#pragma unroll
    for (int nt = 0; nt < D / 8; ++nt) {
      // lanes 0..15 supply the row addresses of the two 8x8 blocks (keys 0-7, keys 8-15) of columns nt*8 .. nt*8+7
      const uint32_t addr = smem_u32(v + (lane & 15) * ld + nt * 8);
      uint32_t b0, b1;
      asm volatile("ldmatrix.sync.aligned.m8n8.x2.trans.shared.b16 {%0, %1}, [%2];" : "=r"(b0), "=r"(b1) : "r"(addr));
      float o[4] = {0.f, 0.f, 0.f, 0.f};
      mma_16816(o, pa, b0, b1);
      *reinterpret_cast<uint32_t*>(orow_lo + nt * 8 + 2 * t) = pack_f16x2(o[0], o[1]);
      *reinterpret_cast<uint32_t*>(orow_hi + nt * 8 + 2 * t) = pack_f16x2(o[2], o[3]);
    }
  }
  __syncthreads();
  __half* obase = out + pix * 16 * ldo + hb0 * D;
  for (int i = threadIdx.x; i < 16 * vseg; i += blockDim.x) {
    const int f = i / vseg, vv = i % vseg;
    *reinterpret_cast<uint4*>(obase + (int64_t)f * ldo + vv * 8) = *reinterpret_cast<const uint4*>(sm + f * ld + vv * 8);
  }
}

// ------------------------------------------------------------------------------------------------ misc elementwise
__global__ void upsample2x_kernel(const __half* __restrict__ x, __half* __restrict__ y, int64_t n, int h, int w, int c) {
  const int vec = c / 8;
  const int64_t total = n * (2 * h) * (2 * w) * vec;
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int v = (int)(idx % vec);
  const int64_t pix = idx / vec;
  const int ox = (int)(pix % (2 * w));
  const int oy = (int)((pix / (2 * w)) % (2 * h));
  const int64_t img = pix / ((int64_t)4 * h * w);
  const uint4 val = __ldg(reinterpret_cast<const uint4*>(x + ((img * h + oy / 2) * w + ox / 2) * c) + v);
  *(reinterpret_cast<uint4*>(y + pix * c) + v) = val;
}

__global__ void silu_rows_kernel(const float* __restrict__ x, __half* __restrict__ y, int64_t rows, int c, int rep) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= rows * c) return;
  const int64_t r = idx / c;
  const int j = (int)(idx % c);
  y[idx] = __float2half_rn(silu_f(x[(r / rep) * c + j]));
}

__global__ void timestep_proj_kernel(const float* __restrict__ t, float* __restrict__ out, int rows, int half) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= rows * half) return;
  const int r = idx / half, i = idx % half;
  const float freq = expf(-9.210340371976184f * (float)i / (float)half);   // ln(10000)
  const float e = t[r] * freq;
  out[r * 2 * half + i] = cosf(e);           // flip_sin_to_cos=True -> [cos | sin]
  out[r * 2 * half + half + i] = sinf(e);
}

__global__ void linear_f32_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ b,
                                  float* __restrict__ y, int m, int n, int k, int act_in, int accumulate) {
  // one warp per output element
  const int64_t wid = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (wid >= (int64_t)m * n) return;
  const int r = (int)(wid / n), j = (int)(wid % n);
  float acc = 0.f;
  for (int i = lane; i < k; i += 32) {
    float xv = x[(int64_t)r * k + i];
    if (act_in == 1) xv = silu_f(xv);
    acc += xv * w[(int64_t)j * k + i];
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if (lane == 0) {
    if (b) acc += b[j];
    if (accumulate) acc += y[(int64_t)r * n + j];
    y[(int64_t)r * n + j] = acc;
  }
}

__global__ void cast_f32_f16_kernel(const float* __restrict__ x, __half* __restrict__ y, int64_t n) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx < n) y[idx] = __float2half_rn(x[idx]);
}

// conv_in: sample [BN, Cin, F, H, W] fp32 -> y NHWC fp16 [(BN F) H W, Cout].  Lanes = consecutive pixels (coalesced input
// reads), a thread produces 16 output channels (one full 32-byte sector): its Cin*9 inputs sit in registers, the weights of
// the block's channel slice in shared memory as [cin*9][16] (all lanes read the same address -> broadcast).
constexpr int kConvInMaxK = 72;   // cin * 9 <= 72 (cin <= 8)
__global__ void __launch_bounds__(128)
conv_in_kernel(const float* __restrict__ sample, const float* __restrict__ w, const float* __restrict__ b, __half* __restrict__ y,
               int bn, int cin, int f, int h, int wd, int cout) {
  __shared__ __align__(16) float sw[kConvInMaxK * 16];
  __shared__ float sb[16];
  const int co0 = blockIdx.y * 16;
  const int kk = cin * 9;
  for (int i = threadIdx.x; i < kk * 16; i += blockDim.x) {
    const int k = i / 16, o = i % 16;                       // k = ci * 9 + tap
    sw[i] = (co0 + o < cout) ? w[(int64_t)(co0 + o) * kk + k] : 0.f;
  }
  if (threadIdx.x < 16) sb[threadIdx.x] = (co0 + threadIdx.x < cout) ? b[co0 + threadIdx.x] : 0.f;
  __syncthreads();
  const int64_t pix = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t npix = (int64_t)bn * f * h * wd;
  if (pix >= npix) return;
  const int x = (int)(pix % wd), yy = (int)((pix / wd) % h);
  const int fr = (int)((pix / ((int64_t)wd * h)) % f);
  const int smp = (int)(pix / ((int64_t)wd * h * f));
  float acc[16];
#pragma unroll
  for (int o = 0; o < 16; ++o) acc[o] = sb[o];
  for (int ci = 0; ci < cin; ++ci) {
    const float* img = sample + (((int64_t)smp * cin + ci) * f + fr) * h * wd;
#pragma unroll
    for (int tap = 0; tap < 9; ++tap) {
      const int iy = yy + tap / 3 - 1, ix = x + tap % 3 - 1;
      const float v = (iy >= 0 && iy < h && ix >= 0 && ix < wd) ? __ldg(img + iy * wd + ix) : 0.f;
      const float4* wr = reinterpret_cast<const float4*>(sw + (ci * 9 + tap) * 16);
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const float4 ww = wr[q];
        acc[4 * q] = fmaf(v, ww.x, acc[4 * q]); acc[4 * q + 1] = fmaf(v, ww.y, acc[4 * q + 1]);
        acc[4 * q + 2] = fmaf(v, ww.z, acc[4 * q + 2]); acc[4 * q + 3] = fmaf(v, ww.w, acc[4 * q + 3]);
      }
    }
  }
  uint32_t hw8[8];     // cout % 16 == 0 (checked on the host): one full 32-byte sector per thread
#pragma unroll
  for (int i = 0; i < 8; ++i) hw8[i] = pack_f16x2(acc[2 * i], acc[2 * i + 1]);
  st_global_256(y + pix * cout + co0, hw8);
}

// conv_out: x NHWC fp16 [(BN F) H W, Cin] -> y [BN, Cout, F, H, W] fp32, cout <= 4.  Four lanes per pixel split the input
// channels in 16-byte vectors (vector c, c+4, ...); weights transposed into shared memory as [tap][cin][4] once per block.
__global__ void __launch_bounds__(256)
conv_out_kernel(const __half* __restrict__ x, const float* __restrict__ w, const float* __restrict__ b, float* __restrict__ y,
                int bn, int cin, int f, int h, int wd, int cout) {
  // [tap][part][channels of that part][4 couts] + one float4 of padding per (tap, part): the four lanes of a pixel read
  // different parts at the same time, the padding puts them on different banks
  extern __shared__ __align__(16) float swo[];
  const int nvec = cin / 8;
  const int vpp = (nvec + 3) / 4;                           // 16-byte vectors per part
  const int pstride = (vpp * 8 + 1) * 4;                    // floats per (tap, part) block
  for (int i = threadIdx.x; i < 9 * cin * 4; i += blockDim.x) {
    const int o = i & 3, c = (i >> 2) % cin, tap = (i >> 2) / cin;
    const int vb = c >> 3, prt = vb & 3, loc = (vb >> 2) * 8 + (c & 7);
    swo[(tap * 4 + prt) * pstride + loc * 4 + o] = o < cout ? w[((int64_t)o * cin + c) * 9 + tap] : 0.f;
  }
  __syncthreads();
  const int64_t gid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t pix = gid >> 2;
  const int part = (int)(gid & 3);
  const int64_t npix = (int64_t)bn * f * h * wd;
  const bool ok = pix < npix;
  const int px = ok ? (int)(pix % wd) : 0, py = ok ? (int)((pix / wd) % h) : 0;
  const int64_t img = ok ? pix / ((int64_t)wd * h) : 0;   // (bn f)
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
  if (ok) {
    for (int tap = 0; tap < 9; ++tap) {
      const int iy = py + tap / 3 - 1, ix = px + tap % 3 - 1;
      if (iy < 0 || iy >= h || ix < 0 || ix >= wd) continue;
      const uint4* src = reinterpret_cast<const uint4*>(x + ((img * h + iy) * wd + ix) * cin);
      const float4* wt = reinterpret_cast<const float4*>(swo + (size_t)(tap * 4 + part) * pstride);
      for (int vb = part, j = 0; vb < nvec; vb += 4, ++j) {
        const uint4 v = __ldg(src + vb);
        const __half2* hv = reinterpret_cast<const __half2*>(&v);
#pragma unroll
        for (int t = 0; t < 4; ++t) {
          const float2 fv = __half22float2(hv[t]);
          const float4 w0 = wt[j * 8 + 2 * t], w1 = wt[j * 8 + 2 * t + 1];
          acc[0] = fmaf(fv.x, w0.x, fmaf(fv.y, w1.x, acc[0]));
          acc[1] = fmaf(fv.x, w0.y, fmaf(fv.y, w1.y, acc[1]));
          acc[2] = fmaf(fv.x, w0.z, fmaf(fv.y, w1.z, acc[2]));
          acc[3] = fmaf(fv.x, w0.w, fmaf(fv.y, w1.w, acc[3]));
        }
      }
    }
  }
#pragma unroll
  for (int o = 0; o < 4; ++o) {
    acc[o] += __shfl_xor_sync(0xffffffffu, acc[o], 1);
    acc[o] += __shfl_xor_sync(0xffffffffu, acc[o], 2);
  }
  if (ok && part < cout) {     // lane `part` of the pixel's quad writes output channel `part`
    const int fr = (int)(img % f);
    const int64_t smp = img / f;
    const float val = part == 0 ? acc[0] : part == 1 ? acc[1] : part == 2 ? acc[2] : acc[3];
    y[(((smp * cout + part) * f + fr) * h + py) * wd + px] = val + b[part];
  }
}

// cfg_mode: 0 = noise_pred holds bn samples (no guidance); 1 = (uncond, cond) halves; 2 = (cond, uncond) halves.
// z (variance noise) is read only when non-null.  Both a3d_ddim_step and a3d_ddim_cfg_step launch this kernel.
__global__ void ddim_step_kernel(float* __restrict__ lat, const float* __restrict__ eps_in, const float* __restrict__ first,
                                 const float* __restrict__ z, int bn, int c, int f, int hw, int cfg_mode, float g, float a_t,
                                 float a_prev, float dir_coef, float std_dev) {
  const int64_t n = (int64_t)bn * c * f * hw;
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n) return;
  const int fr = (int)((idx / hw) % f);
  if (fr == 0 && first) {
    const int64_t sc = idx / ((int64_t)f * hw);  // (bn c)
    lat[idx] = first[sc * hw + idx % hw];
    return;
  }
  float eps;
  if (cfg_mode == 0) {
    eps = eps_in[idx];
  } else {
    const float e0 = eps_in[idx], e1 = eps_in[n + idx];
    eps = cfg_mode == 1 ? (e0 + g * (e1 - e0)) : (e0 + g * (e0 - e1));
  }
  const float x = lat[idx];
  const float x0 = (x - sqrtf(1.f - a_t) * eps) / sqrtf(a_t);
  float v = sqrtf(a_prev) * x0 + dir_coef * eps;
  if (z) v += std_dev * z[idx];
  lat[idx] = v;
}

// a3d_sampler_step: the per-element order of operations is written above the declaration in include/a3d.h.
__global__ void sampler_step_kernel(a3d_sampler_step_args a) {
  const int64_t n = (int64_t)a.bn * a.c * a.f * a.hw;
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= n) return;
  if (a.first_frame && (int)((idx / a.hw) % a.f) == 0) {
    const int64_t sc = idx / ((int64_t)a.f * a.hw);  // (bn c)
    a.latents[idx] = a.first_frame[sc * a.hw + idx % a.hw];
    return;
  }
  float eps;
  if (a.cfg_mode == 0) {
    eps = a.noise_pred[idx];
  } else {
    const float e0 = a.noise_pred[idx], e1 = a.noise_pred[n + idx];
    eps = a.cfg_mode == 1 ? (e0 + a.guidance * (e1 - e0)) : (e0 + a.guidance * (e0 - e1));
  }
  const float x = a.latents[idx];
  float v;
  if (a.kind == A3D_SAMPLER_DPMPP) {
    const float m0 = (x - a.sigma_s0 * eps) / a.alpha_s0;
    if (a.history_out) a.history_out[idx] = m0;
    v = a.c_x * x - a.c_m0 * m0;
    if (a.order == 2) v += a.c_d1 * (a.inv_r0 * (m0 - a.history_in[idx]));
  } else {
    const float x0 = x - a.sigma * eps;
    const float d = (x - x0) / a.sigma;
    v = x + d * a.dt;
    if (a.sigma_up != 0.f) v += a.noise[idx] * a.sigma_up;
  }
  a.latents[idx] = v;
}

}  // namespace a3d

using namespace a3d;

static void gn_geometry(int C, int64_t samples, int64_t rows_per_sample, int* rows_par, int* threads, int* chunk_rows, int* chunks) {
  const int vpr = C / 8;
  int rp = 256 / vpr;
  if (rp < 1) rp = 1;
  *rows_par = rp;
  *threads = ((rp * vpr + 31) / 32) * 32;   // <= 256 (C / 8 <= 160 for the UNet's widths) or one row per block
  int cr = 128;
  const int64_t fill = 4 * (int64_t)sm_count();   // blocks for about four waves per SM
  while (cr > 4 * rp && ((rows_per_sample + cr - 1) / cr) * samples < fill) cr /= 2;
  *chunk_rows = cr;
  *chunks = (int)((rows_per_sample + cr - 1) / cr);
}

extern "C" size_t a3d_group_norm_ws_bytes(int64_t samples, int64_t rows_per_sample, int c, int groups) {
  if (c < 8 || samples < 1 || rows_per_sample < 1 || groups < 1) return 0;
  int rows_par, threads, chunk_rows, chunks;
  gn_geometry(c, samples, rows_per_sample, &rows_par, &threads, &chunk_rows, &chunks);
  return sizeof(float) * ((size_t)2 * groups * samples + (size_t)3 * groups * samples * chunks);
}

extern "C" int a3d_group_norm(const void* x1, int c1, const void* x2, int c2, const float* gamma, const float* beta, void* y,
                              int64_t samples, int64_t rows_per_sample, int groups, float eps, int silu, int64_t perm_a,
                              int64_t perm_b, float* ws_stats, void* stream) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int C = c1 + (x2 ? c2 : 0);
  if (!x2) c2 = 0;
  if (C % groups || C % 8 || c1 % 8 || c2 % 8 || C / 8 > 1024 || groups > 64)
    return fail(A3D_EINVAL, "a3d_group_norm: unsupported channels C=%d (c1=%d c2=%d) groups=%d", C, c1, c2, groups);
  if (rows_per_sample > (int64_t)1 << 30 || samples > 65535) return fail(A3D_EINVAL, "a3d_group_norm: extent too large");
  const int vpr = C / 8;
  int rows_par, threads, chunk_rows, chunks;
  gn_geometry(C, samples, rows_per_sample, &rows_par, &threads, &chunk_rows, &chunks);
  if (threads > 512) return fail(A3D_EINVAL, "a3d_group_norm: C=%d too wide", C);
  const size_t smem = (size_t)rows_par * vpr * 6 * sizeof(float);
  if (smem > 48 * 1024) return fail(A3D_EINVAL, "a3d_group_norm: C=%d needs %zu B of shared memory", C, smem);
  float* stats = ws_stats;                                          // [samples][groups][mean, rstd]
  float* partials = ws_stats + 2 * (size_t)groups * samples;         // [samples][chunks][groups][n, mean, M2]
  dim3 grid((unsigned)chunks, (unsigned)samples);
  gn_stats_kernel<<<grid, threads, smem, st>>>(reinterpret_cast<const __half*>(x1), c1, reinterpret_cast<const __half*>(x2), c2,
                                               (int)rows_per_sample, groups, rows_par, chunk_rows, partials);
  A3D_LAUNCH_CHECK();
  gn_finalize_kernel<<<dim3((groups + 7) / 8, (unsigned)samples), 256, 0, st>>>(partials, chunks, groups, eps, stats);
  A3D_LAUNCH_CHECK();
  gn_apply_kernel<<<grid, threads, 0, st>>>(reinterpret_cast<const __half*>(x1), c1, reinterpret_cast<const __half*>(x2), c2,
                                            gamma, beta, reinterpret_cast<__half*>(y), (int)rows_per_sample, groups, eps, silu,
                                            perm_a, perm_b, rows_par, chunk_rows, stats);
  A3D_LAUNCH_CHECK();
  return A3D_OK;
}

extern "C" int a3d_group_norm_backward(const void* x, int c, const float* gamma, const float* beta, const float* fwd_ws_stats,
                                       const void* dy, void* dx, int64_t samples, int64_t rows_per_sample, int groups, int silu,
                                       float* ws, void* stream) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (c % groups || c % 8 || c / 8 > 1024 || groups > 64) return fail(A3D_EINVAL, "a3d_group_norm_backward: unsupported channels %d", c);
  if (!x || !dy || !dx || !fwd_ws_stats || !ws) return fail(A3D_EINVAL, "a3d_group_norm_backward: null operand");
  if (rows_per_sample > (int64_t)1 << 30 || samples > 65535) return fail(A3D_EINVAL, "a3d_group_norm_backward: extent too large");
  const int vpr = c / 8;
  int rows_par, threads, chunk_rows, chunks;
  gn_geometry(c, samples, rows_per_sample, &rows_par, &threads, &chunk_rows, &chunks);
  if (threads > 512) return fail(A3D_EINVAL, "a3d_group_norm_backward: C=%d too wide", c);
  const size_t smem = (size_t)rows_par * vpr * 4 * sizeof(float);
  float* sums = ws;                                           // [samples][groups][mean g, mean g*xhat]
  float* partials = ws + 2 * (size_t)groups * samples;        // [samples][chunks][groups][2]   (fits a3d_group_norm_ws_bytes)
  dim3 grid((unsigned)chunks, (unsigned)samples);
  const __half* xh = reinterpret_cast<const __half*>(x);
  const __half* dyh = reinterpret_cast<const __half*>(dy);
  gn_bwd_kernel<false><<<grid, threads, smem, st>>>(xh, dyh, gamma, beta, fwd_ws_stats, nullptr, partials, nullptr, c, (int)rows_per_sample,
                                                    groups, silu, rows_par, chunk_rows);
  A3D_LAUNCH_CHECK();
  const float inv_n = 1.0f / ((float)rows_per_sample * (float)(c / groups));
  gn_bwd_finalize_kernel<<<dim3((groups + 7) / 8, (unsigned)samples), 256, 0, st>>>(partials, chunks, groups, inv_n, sums);
  A3D_LAUNCH_CHECK();
  gn_bwd_kernel<true><<<grid, threads, 0, st>>>(xh, dyh, gamma, beta, fwd_ws_stats, sums, nullptr, reinterpret_cast<__half*>(dx), c,
                                                (int)rows_per_sample, groups, silu, rows_par, chunk_rows);
  A3D_LAUNCH_CHECK();
  return A3D_OK;
}

extern "C" int a3d_layer_norm(const void* x, const float* gamma, const float* beta, void* y, int64_t rows, int c, float eps,
                              void* stream) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (c % 8 || c > 1280) return fail(A3D_EINVAL, "a3d_layer_norm: C=%d must be a multiple of 8 and <= 1280", c);
  const __half* xi = reinterpret_cast<const __half*>(x);
  __half* yo = reinterpret_cast<__half*>(y);
  const int warps = 4;
  if (c == 320) {
    layer_norm_kernel<8><<<(unsigned)((rows + warps * 4 - 1) / (warps * 4)), warps * 32, 0, st>>>(xi, gamma, beta, yo, rows, eps);
  } else if (c == 640) {
    layer_norm_kernel<16><<<(unsigned)((rows + warps * 2 - 1) / (warps * 2)), warps * 32, 0, st>>>(xi, gamma, beta, yo, rows, eps);
  } else if (c == 1280) {
    layer_norm_kernel<32><<<(unsigned)((rows + warps - 1) / warps), warps * 32, 0, st>>>(xi, gamma, beta, yo, rows, eps);
  } else {
    layer_norm_generic_kernel<<<(unsigned)((rows + 7) / 8), 256, 0, st>>>(xi, gamma, beta, yo, rows, c, eps);
  }
  A3D_LAUNCH_CHECK();
  return A3D_OK;
}

// The checks of a3d_temporal_attn and its kernel: temporal_attn16_kernel (16 frames, HB = 320 / d heads per block) or the
// generic one.  *ldo: the output row stride, 0 resolved to heads * d.
static int plan_temporal(const void* out, int frames, int heads, int d, int64_t* ldo, bool* frames16) {
  if (frames > 32 || frames * heads > 1024) return fail(A3D_EINVAL, "a3d_temporal_attn: frames=%d heads=%d", frames, heads);
  if (*ldo == 0) *ldo = (int64_t)heads * d;
  if (*ldo < (int64_t)heads * d || *ldo % 8 || (reinterpret_cast<uintptr_t>(out) & 15))
    return fail(A3D_EINVAL, "a3d_temporal_attn: output row stride %lld must be >= C, a multiple of 8, 16-byte aligned base",
                (long long)*ldo);
  if (d != 40 && d != 80 && d != 160) return fail(A3D_EINVAL, "a3d_temporal_attn: head dim %d not in {40,80,160}", d);
  const int hb = 320 / d;
  *frames16 = frames == 16 && heads % hb == 0 && heads / hb <= 65535;
  return A3D_OK;
}

template <int D>
static int launch_temporal(const void* qkv, void* out, int64_t pixels, int frames, int heads, float scale, int64_t ldo,
                           bool frames16, cudaStream_t st) {
  constexpr int HB = 320 / D;   // 8 / 4 / 2 heads per block
  if (frames16) {
    const size_t smem16 = (size_t)16 * (3 * HB * D + 8) * 2;   // 31 KB
    temporal_attn16_kernel<D, HB><<<dim3((unsigned)pixels, (unsigned)(heads / HB)), HB * 32, smem16, st>>>(
        reinterpret_cast<const __half*>(qkv), reinterpret_cast<__half*>(out), heads, scale * 1.4426950408889634f, ldo);
    A3D_LAUNCH_CHECK();
    return A3D_OK;
  }
  const size_t smem = (size_t)frames * 2 * heads * D * 2;
  static size_t max_set = 0;
  if (smem > 48 * 1024 && smem > max_set) {
    A3D_CUDA_CHECK(cudaFuncSetAttribute(temporal_attn_kernel<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    max_set = smem;
  }
  const int threads = ((frames * heads + 31) / 32) * 32;
  temporal_attn_kernel<D><<<(unsigned)pixels, threads, smem, st>>>(reinterpret_cast<const __half*>(qkv), reinterpret_cast<__half*>(out),
                                                                   frames, heads, scale, ldo);
  A3D_LAUNCH_CHECK();
  return A3D_OK;
}

extern "C" int a3d_temporal_attn_kernel(const void* out, int64_t pixels, int frames, int heads, int d, int64_t ldo, char* name,
                                        size_t n) {
  bool frames16;
  if (int r = plan_temporal(out, frames, heads, d, &ldo, &frames16)) return r;
  return kernel_name(name, n, "%s", frames16 ? "frames16" : "generic");
}

extern "C" int a3d_temporal_attn(const void* qkv, void* out, int64_t pixels, int frames, int heads, int d, float scale,
                                 int64_t ldo, void* stream) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  bool frames16;
  if (int r = plan_temporal(out, frames, heads, d, &ldo, &frames16)) return r;
  switch (d) {
    case 40: return launch_temporal<40>(qkv, out, pixels, frames, heads, scale, ldo, frames16, st);
    case 80: return launch_temporal<80>(qkv, out, pixels, frames, heads, scale, ldo, frames16, st);
    default: return launch_temporal<160>(qkv, out, pixels, frames, heads, scale, ldo, frames16, st);
  }
}

extern "C" int a3d_upsample2x(const void* x, void* y, int64_t n, int h, int w, int c, void* stream) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (c % 8) return fail(A3D_EINVAL, "a3d_upsample2x: C %% 8");
  const int64_t total = n * 4 * h * w * (c / 8);
  upsample2x_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(reinterpret_cast<const __half*>(x),
                                                                    reinterpret_cast<__half*>(y), n, h, w, c);
  A3D_LAUNCH_CHECK();
  return A3D_OK;
}

extern "C" int a3d_silu_rows(const float* x, void* y, int64_t rows, int c, int rep, void* stream) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int64_t total = rows * c;
  silu_rows_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(x, reinterpret_cast<__half*>(y), rows, c, rep);
  A3D_LAUNCH_CHECK();
  return A3D_OK;
}

extern "C" int a3d_conv_in(const float* sample, const float* w, const float* b, void* y, int bn, int cin, int f, int h,
                           int wd, int cout, void* stream) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (cin * 9 > kConvInMaxK) return fail(A3D_EINVAL, "a3d_conv_in: cin <= 8 (got %d)", cin);
  if (cout % 16 || (reinterpret_cast<uintptr_t>(y) & 31)) return fail(A3D_EINVAL, "a3d_conv_in: cout %% 16 and 32-byte aligned output");
  const int64_t npix = (int64_t)bn * f * h * wd;
  dim3 grid((unsigned)((npix + 127) / 128), (unsigned)(cout / 16));
  conv_in_kernel<<<grid, 128, 0, st>>>(sample, w, b, reinterpret_cast<__half*>(y), bn, cin, f, h, wd, cout);
  A3D_LAUNCH_CHECK();
  return A3D_OK;
}

extern "C" int a3d_conv_out(const void* x, const float* w, const float* b, float* y, int bn, int cin, int f, int h, int wd,
                            int cout, void* stream) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (cout > 4 || cin % 8) return fail(A3D_EINVAL, "a3d_conv_out: cout <= 4 and cin %% 8 == 0 (got %d, %d)", cout, cin);
  const int64_t npix = (int64_t)bn * f * h * wd;
  const int vpp = (cin / 8 + 3) / 4;
  const size_t smem = (size_t)9 * 4 * (vpp * 8 + 1) * 4 * sizeof(float);
  static size_t max_set = 0;
  if (smem > 48 * 1024 && smem > max_set) {
    A3D_CUDA_CHECK(cudaFuncSetAttribute(conv_out_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    max_set = smem;
  }
  conv_out_kernel<<<(unsigned)((npix * 4 + 255) / 256), 256, smem, st>>>(reinterpret_cast<const __half*>(x), w, b, y, bn, cin, f, h,
                                                                        wd, cout);
  A3D_LAUNCH_CHECK();
  return A3D_OK;
}

extern "C" int a3d_timestep_proj(const float* t, float* out, int rows, int half, void* stream) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  timestep_proj_kernel<<<(rows * half + 127) / 128, 128, 0, st>>>(t, out, rows, half);
  A3D_LAUNCH_CHECK();
  return A3D_OK;
}

extern "C" int a3d_linear_f32(const float* x, const float* w, const float* b, float* y, int m, int n, int k, int act_in,
                              int accumulate, void* stream) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int64_t threads = (int64_t)m * n * 32;
  linear_f32_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, st>>>(x, w, b, y, m, n, k, act_in, accumulate);
  A3D_LAUNCH_CHECK();
  return A3D_OK;
}

extern "C" int a3d_cast_f32_f16(const float* x, void* y, int64_t n, void* stream) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  cast_f32_f16_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(x, reinterpret_cast<__half*>(y), n);
  A3D_LAUNCH_CHECK();
  return A3D_OK;
}

extern "C" int a3d_ddim_step(float* latents, const float* noise_pred, const float* first_frame, const float* variance_noise,
                             int bn, int c, int f, int hw, int cfg_mode, float guidance, float alpha_t, float alpha_prev,
                             float dir_coef, float std_dev, void* stream) {
  if (cfg_mode < 0 || cfg_mode > 2) return fail(A3D_EINVAL, "a3d_ddim_step: cfg_mode %d is not 0, 1 or 2", cfg_mode);
  if (std_dev != 0.f && !variance_noise) return fail(A3D_EINVAL, "a3d_ddim_step: std_dev %g needs variance_noise", std_dev);
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int64_t n = (int64_t)bn * c * f * hw;
  ddim_step_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(latents, noise_pred, first_frame, variance_noise, bn, c, f, hw,
                                                               cfg_mode, guidance, alpha_t, alpha_prev, dir_coef, std_dev);
  A3D_LAUNCH_CHECK();
  return A3D_OK;
}

extern "C" int a3d_ddim_cfg_step(float* latents, const float* noise_pred, const float* first_frame, int bn, int c, int f,
                                 int hw, float guidance, float alpha_t, float alpha_prev, int uncond_first, void* stream) {
  return a3d_ddim_step(latents, noise_pred, first_frame, nullptr, bn, c, f, hw, uncond_first ? 1 : 2, guidance, alpha_t,
                       alpha_prev, sqrtf(1.f - alpha_prev), 0.f, stream);
}

extern "C" int a3d_sampler_step(const a3d_sampler_step_args* args, void* stream) {
  if (!args) return fail(A3D_EINVAL, "a3d_sampler_step: args is NULL");
  const a3d_sampler_step_args& a = *args;
  if (a.kind != A3D_SAMPLER_DPMPP && a.kind != A3D_SAMPLER_EULER)
    return fail(A3D_EINVAL, "a3d_sampler_step: kind %d is not A3D_SAMPLER_DPMPP (0) or A3D_SAMPLER_EULER (1)", a.kind);
  if (a.cfg_mode < 0 || a.cfg_mode > 2) return fail(A3D_EINVAL, "a3d_sampler_step: cfg_mode %d is not 0, 1 or 2", a.cfg_mode);
  if (a.kind == A3D_SAMPLER_DPMPP && a.order != 1 && a.order != 2)
    return fail(A3D_EINVAL, "a3d_sampler_step: DPM-Solver++ order %d is not 1 or 2", a.order);
  if (a.kind == A3D_SAMPLER_DPMPP && a.order == 2 && !a.history_in)
    return fail(A3D_EINVAL, "a3d_sampler_step: order 2 needs history_in (the previous step's m0)");
  if (a.kind == A3D_SAMPLER_EULER && a.sigma_up != 0.f && !a.noise)
    return fail(A3D_EINVAL, "a3d_sampler_step: sigma_up %g needs noise", a.sigma_up);
  if (!a.latents || !a.noise_pred) return fail(A3D_EINVAL, "a3d_sampler_step: latents and noise_pred are required");
  const int64_t n = (int64_t)a.bn * a.c * a.f * a.hw;
  if (n <= 0) return A3D_OK;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  sampler_step_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(a);
  A3D_LAUNCH_CHECK();
  return A3D_OK;
}
