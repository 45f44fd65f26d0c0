// a3d_attention: O = softmax(scale * Q K^T) V, flash-style, on Hopper tensor cores (wgmma).
//
//   one CTA = one 128-row query tile of one (batch, head); 9 warps:
//     warp 8      TMA producer (Q once, K/V tiles of 64 keys through a ring of smem stages; 128B-swizzled boxes read straight
//                 out of the projection GEMM's output through rank-5 strided views -> the reference's
//                 "(b n f) l c -> (b f) (n l) c" regroupings and frame-0 K/V broadcasts never materialise)
//     warps 0..7  two consumer warpgroups of 64 query rows each:  S = Q K^T (wgmma, both operands K-major in smem, fp32 in
//                 registers), online softmax in registers, O += P V (wgmma with P as the register A operand, V MN-major)
//   Single-pass ("stale stabiliser") softmax: the running row maximum of the previous key steps stays the exponent offset
//   and O is rescaled only when a later step raises it by more than kRescaleLog2 (P then stays below 2^kRescaleLog2, far
//   inside fp16).  The row sum is not computed separately: V carries a column of ones at index d (placed there by the
//   projection epilogue), so O[:, d] accumulates sum(P) in fp32 alongside the PV product.
//
// Replaces xformers.ops.memory_efficient_attention at animatediff/models/attention_processor.py:103,233,268,405,416,656,691.
#include <stdlib.h>

#include <type_traits>

#include "a3d_common.cuh"
#include "a3d_host.cuh"
#include "a3d_wgmma.cuh"

namespace a3d {

struct AttnDev {
  int q_tiles, kv_tiles;
  int rows_q, rows_k;            // valid rows per q tile (<= 128) / in the LAST kv tile (<= 64)
  int heads;
  int q_t1, q_box1, q_box2, q_e1, q_e3;   // q_e1: rows at or past it belong to the next batch (ragged last query tile)
  int k_t1, k_box1, k_box2, k_e3, kv_div, kv_i3_zero;
  uint32_t q_box_bytes, k_box_bytes;   // bytes one 64-column TMA box delivers
  float scale_log2;
  __half* out;
  int64_t os1, os2, os3, os4;
  int accumulate;
  float out_scale;
  unsigned long long* dbg;   // debug (null in production): dbg[0] counts (warp, step) pairs that took the lazy-rescale branch
};

constexpr float kRescaleLog2 = 8.0f;
constexpr int kAttnThreads = 288;

template <int D>
struct AttnCfg {
  static constexpr int kDqk = (D + 15) / 16 * 16;        // 48 / 80 / 160
  static constexpr int kDv = (D + 1 + 15) / 16 * 16;     // 48 / 96 / 176
  static constexpr int kQB = (kDqk + 63) / 64;           // 64-column boxes per Q / K row: 1 / 2 / 3
  static constexpr int kVB = (kDv + 63) / 64;            // 1 / 2 / 3
  static constexpr int kStages = (D == 160) ? 3 : 4;
  static constexpr int kQBox = 128 * 128;                // 128 rows x 64 cols fp16
  static constexpr int kKVBox = 64 * 128;                // 64 keys x 64 cols fp16
  static constexpr int kSmemQ = kQB * kQBox;
  static constexpr int kSmemK = kStages * kQB * kKVBox;
  static constexpr int kSmemV = kStages * kVB * kKVBox;
  static constexpr int kSmemBytes = kSmemQ + kSmemK + kSmemV + 1024 + 256;
  static constexpr int kMinBlocks = (kSmemBytes <= 113 * 1024) ? 2 : 1;
  static_assert(kSmemBytes <= 227 * 1024, "shared memory budget");
};

// f(integral_constant<I>), f(integral_constant<I + 1>), ... up to N - 1, while f returns true
template <int I, int N, class F>
__device__ __forceinline__ void static_for(F&& f) {
  if constexpr (I < N) {
    if (f(std::integral_constant<int, I>{})) static_for<I + 1, N>(f);
  }
}

template <int N>
__device__ __forceinline__ void wgmma_pv(float (&o)[N / 2], const uint32_t (&a)[4], uint64_t bdesc, uint32_t acc) {
  if constexpr (N == 48) wgmma_rs_n48<1>(o, a, bdesc, acc);
  else if constexpr (N == 96) wgmma_rs_n96<1>(o, a, bdesc, acc);
  else wgmma_rs_n176<1>(o, a, bdesc, acc);
}

template <int D>
__global__ void __launch_bounds__(kAttnThreads, AttnCfg<D>::kMinBlocks)
attn_tc_kernel(const AttnDev p, const __grid_constant__ CUtensorMap mapQ, const __grid_constant__ CUtensorMap mapK,
               const __grid_constant__ CUtensorMap mapV) {
  using Cfg = AttnCfg<D>;
  constexpr int S = Cfg::kStages;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sQ = smem;
  uint8_t* sK = sQ + Cfg::kSmemQ;
  uint8_t* sV = sK + Cfg::kSmemK;
  uint64_t* bars = reinterpret_cast<uint64_t*>(sV + Cfg::kSmemV);
  uint64_t* q_full = bars;
  uint64_t* k_full = bars + 1;          // [S]
  uint64_t* v_full = k_full + S;        // [S]
  uint64_t* kv_empty = v_full + S;      // [S]

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int qt = blockIdx.x;
  const int head = blockIdx.y;
  const int qb = blockIdx.z;
  const int n = p.kv_tiles;
  const int rows_tile = p.k_box1 * p.k_box2;

  if (p.rows_q < 128 || rows_tile < 64) {
    // partially filled tiles: rows TMA never writes must read as zeros (0 * garbage could be NaN in P V)
    uint4* z = reinterpret_cast<uint4*>(sQ);
    const int n16 = (Cfg::kSmemQ + Cfg::kSmemK + Cfg::kSmemV) / 16;
    for (int i = threadIdx.x; i < n16; i += blockDim.x) z[i] = make_uint4(0, 0, 0, 0);
    fence_proxy_async_smem();
  }
  if (warp == 8 && lane == 0) {
    tma_prefetch_desc(&mapQ);
    tma_prefetch_desc(&mapK);
    tma_prefetch_desc(&mapV);
    mbar_init(q_full, 1);
    for (int i = 0; i < S; ++i) {
      mbar_init(&k_full[i], 1);
      mbar_init(&v_full[i], 1);
      mbar_init(&kv_empty[i], 8);   // one arrive per consumer warp
    }
    mbar_fence_init();
  }
  __syncthreads();

  const int q_i1 = (qt % p.q_t1) * p.q_box1;
  const int q_i2 = (qt / p.q_t1) * p.q_box2;
  const int q_i3 = qb % p.q_e3;
  const int q_i4 = qb / p.q_e3;

  if (warp == 8) {
    // ------------------------------------------------------------------ TMA producer (one thread)
    if (lane == 0) {
      const int kb = qb / p.kv_div;
      const int k_i3 = p.kv_i3_zero ? 0 : (kb % p.k_e3);
      const int k_i4 = kb / p.k_e3;
      mbar_expect_tx(q_full, p.q_box_bytes * Cfg::kQB);
#pragma unroll
      for (int b = 0; b < Cfg::kQB; ++b)
        tma_load_5d(sQ + b * Cfg::kQBox, &mapQ, q_full, head * Cfg::kDqk + b * 64, q_i1, q_i2, q_i3, q_i4);
      for (int j = 0; j < n; ++j) {
        const int st = j % S;
        const int k_i1 = (j % p.k_t1) * p.k_box1, k_i2 = (j / p.k_t1) * p.k_box2;
        mbar_wait(&kv_empty[st], ((j / S) & 1) ^ 1);
        mbar_expect_tx(&k_full[st], p.k_box_bytes * Cfg::kQB);
#pragma unroll
        for (int b = 0; b < Cfg::kQB; ++b)
          tma_load_5d(sK + (st * Cfg::kQB + b) * Cfg::kKVBox, &mapK, &k_full[st], head * Cfg::kDqk + b * 64, k_i1, k_i2, k_i3,
                      k_i4);
        mbar_expect_tx(&v_full[st], p.k_box_bytes * Cfg::kVB);
#pragma unroll
        for (int b = 0; b < Cfg::kVB; ++b)
          tma_load_5d(sV + (st * Cfg::kVB + b) * Cfg::kKVBox, &mapV, &v_full[st], head * Cfg::kDv + b * 64, k_i1, k_i2, k_i3,
                      k_i4);
      }
    }
    return;
  }

  // -------------------------------------------------------------------- consumers: warpgroup wg owns query rows [64 wg, 64 wg + 64)
  // thread (warp w, lane 4 g + t) holds rows r_lo = 16 (w % 4) + g and r_hi = r_lo + 8 of its warpgroup; score / output
  // columns 8 jj + 2 t, +1 (the wgmma accumulator layout)
  //
  // The key loop runs S steps per trip, so the stage of each step is a compile-time constant: every shared-memory
  // descriptor is a base descriptor plus a constant and every barrier address a constant offset.  Only the barrier phase
  // parity flips, once per trip.
  const int wg = warp >> 2;
  const int g = lane >> 2, t = lane & 3;
  float s[32];
  float o[Cfg::kDv / 2];
#pragma unroll
  for (int i = 0; i < Cfg::kDv / 2; ++i) o[i] = 0.f;
  float m_lo = -INFINITY, m_hi = -INFINITY;
  const uint64_t qdesc = make_smem_desc_sw128(smem_u32(sQ + wg * (64 * 128)), 16, 1024);
  const uint64_t kdesc = make_smem_desc_sw128(smem_u32(sK), 16, 1024);
  // V is MN-major: 16 keys = two 8-row swizzle atoms (SBO = 1024 B); the next 64 value columns live one TMA box further
  const uint64_t vdesc = make_smem_desc_sw128(smem_u32(sV), Cfg::kKVBox, 1024);
  // key columns at or past `valid` hold zero fill or the next tile's rows and are masked to -inf: in the last tile, and in
  // every tile when a TMA box holds fewer than 64 keys
  const int mask_from = rows_tile < 64 ? 0 : n - 1;
  uint32_t ph = 0;   // barrier phase of this trip's stages
  mbar_wait(q_full, 0);
  for (int j0 = 0; j0 < n; j0 += S) {
    static_for<0, S>([&](auto stc) {
      constexpr int st = decltype(stc)::value;
      const int j = j0 + st;
      if (j >= n) return false;
      // ---- S = Q K^T
      mbar_wait(&k_full[st], ph);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < Cfg::kDqk / 16; ++kk)
        wgmma_ss_n64<0>(s, desc_add(qdesc, (kk / 4) * Cfg::kQBox + (kk % 4) * 32),
                        desc_add(kdesc, (st * Cfg::kQB + kk / 4) * Cfg::kKVBox + (kk % 4) * 32), kk ? 1u : 0u);
      wgmma_commit();
      wgmma_wait<0>();
      reg_fence(s);
      // ---- row maxima over the valid keys (a quad of lanes shares a row)
      if (j >= mask_from) {
        const int valid = (j == n - 1) ? p.rows_k : rows_tile;
#pragma unroll
        for (int jj = 0; jj < 8; ++jj) {
#pragma unroll
          for (int e = 0; e < 2; ++e)
            if (8 * jj + 2 * t + e >= valid) { s[4 * jj + e] = -INFINITY; s[4 * jj + 2 + e] = -INFINITY; }
        }
      }
      float mx_lo = -INFINITY, mx_hi = -INFINITY;
#pragma unroll
      for (int jj = 0; jj < 8; ++jj) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          mx_lo = fmaxf(mx_lo, s[4 * jj + e]);
          mx_hi = fmaxf(mx_hi, s[4 * jj + 2 + e]);
        }
      }
#pragma unroll
      for (int x = 1; x <= 2; x <<= 1) {
        mx_lo = fmaxf(mx_lo, __shfl_xor_sync(0xffffffffu, mx_lo, x));
        mx_hi = fmaxf(mx_hi, __shfl_xor_sync(0xffffffffu, mx_hi, x));
      }
      const float mn_lo = fmaxf(m_lo, mx_lo * p.scale_log2), mn_hi = fmaxf(m_hi, mx_hi * p.scale_log2);
      if (st == 0 && j == 0) {
        m_lo = mn_lo; m_hi = mn_hi;
      } else if (__any_sync(0xffffffffu, mn_lo - m_lo > kRescaleLog2 || mn_hi - m_hi > kRescaleLog2)) {
        if (p.dbg && lane == 0) atomicAdd(p.dbg, 1ull);
        const float a_lo = ex2_approx(m_lo - mn_lo), a_hi = ex2_approx(m_hi - mn_hi);
#pragma unroll
        for (int c = 0; c < Cfg::kDv / 8; ++c) {
          o[4 * c] *= a_lo; o[4 * c + 1] *= a_lo; o[4 * c + 2] *= a_hi; o[4 * c + 3] *= a_hi;
        }
        m_lo = mn_lo; m_hi = mn_hi;
      }
      // ---- P = exp2(s * scale_log2 - m) -> fp16 A fragments of the four 16-key k-steps
      uint32_t pa[4][4];
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const float* sb = s + 4 * (2 * kk + h);
          pa[kk][2 * h] = pack_f16x2(ex2_approx(fmaf(sb[0], p.scale_log2, -m_lo)), ex2_approx(fmaf(sb[1], p.scale_log2, -m_lo)));
          pa[kk][2 * h + 1] = pack_f16x2(ex2_approx(fmaf(sb[2], p.scale_log2, -m_hi)), ex2_approx(fmaf(sb[3], p.scale_log2, -m_hi)));
        }
      }
      // ---- O += P V
      mbar_wait(&v_full[st], ph);
      wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < 4; ++kk)
        wgmma_pv<Cfg::kDv>(o, pa[kk], desc_add(vdesc, st * Cfg::kVB * Cfg::kKVBox + kk * 2048), 1u);
      wgmma_commit();
      wgmma_wait<0>();
      reg_fence(o);
      __syncwarp();
      if (lane == 0) mbar_arrive(&kv_empty[st]);
      return true;
    });
    ph ^= 1;
  }
  // ---- epilogue: O / O[:, D] -> fp16 -> global (through the query view geometry); column D sits in lane t = 0 of the quad
  const float l_lo = __shfl_sync(0xffffffffu, o[4 * (D / 8)], lane & ~3);
  const float l_hi = __shfl_sync(0xffffffffu, o[4 * (D / 8) + 2], lane & ~3);
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int r = wg * 64 + (warp & 3) * 16 + g + 8 * h;
    const int i1 = q_i1 + r % p.q_box1;
    if (r >= p.rows_q || i1 >= p.q_e1) continue;   // rows TMA zero-filled past e1 are computed but never stored
    const float inv = p.out_scale / (h ? l_hi : l_lo);
    const int i2 = q_i2 + r / p.q_box1;
    __half* orow = p.out + (int64_t)i1 * p.os1 + (int64_t)i2 * p.os2 + (int64_t)q_i3 * p.os3 + (int64_t)q_i4 * p.os4 +
                   head * D + 2 * t;
#pragma unroll
    for (int c = 0; c < D / 8; ++c) {
      float v0 = o[4 * c + 2 * h] * inv, v1 = o[4 * c + 2 * h + 1] * inv;
      if (p.accumulate) {
        const float2 f = __half22float2(*reinterpret_cast<const __half2*>(orow + 8 * c));
        v0 += f.x; v1 += f.y;
      }
      *reinterpret_cast<uint32_t*>(orow + 8 * c) = pack_f16x2(v0, v1);
    }
  }
}

// A strided view as the thread-per-(row, head) kernels read it: element (col, i1, i2, i3, i4) at
// base + col + i1*s1 + i2*s2 + i3*s3 + i4*s4 (a3d_view5 without the column extent)
struct ViewDev {
  const __half* base;
  int64_t s1, s2, s3, s4;
  int e1, e2, e3, e4;
};

// ---------------------------------------------------------------------------------------------------------------
// Few-keys attention (IP-adapter image tokens: 4 keys per image group).  The tensor path would spend a whole CTA
// life-cycle (barrier set-up, TMA round trips) on one 64-key step that is 94% padding; the work itself
// is a read of Q and a read-modify-write of the output.  One thread per (query row, head): fp32 math, 16-byte loads,
// K/V of the image group stay in L1.  HBM-bound: ~(|Q| + 2|out|) bytes.
// ---------------------------------------------------------------------------------------------------------------
constexpr int kFewKeysMax = 8;

template <int D>   // head dim as a template parameter: the channel loops unroll and all Q loads of a row are in flight at once
__global__ void __launch_bounds__(256)
attn_fewkeys_kernel(ViewDev q, ViewDev k, ViewDev v, __half* out, int64_t os1, int64_t os2, int64_t os3, int64_t os4, int heads,
                    int dqk, int dv, float scale_log2, int kv_div, int kv_i3_zero, int accumulate, float out_scale) {
  constexpr int d = D;
  const int Lq = q.e1 * q.e2, Lk = k.e1 * k.e2;
  const int64_t total = (int64_t)q.e3 * q.e4 * Lq * heads;
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int h = (int)(idx % heads);
  const int64_t row = idx / heads;
  const int l = (int)(row % Lq);
  const int qb = (int)(row / Lq);
  const int kb = qb / kv_div;
  const __half* qp = q.base + (int64_t)(l % q.e1) * q.s1 + (int64_t)(l / q.e1) * q.s2 + (int64_t)(qb % q.e3) * q.s3 +
                     (int64_t)(qb / q.e3) * q.s4 + h * dqk;
  const int64_t koff = (int64_t)(kv_i3_zero ? 0 : kb % k.e3) * k.s3 + (int64_t)(kb / k.e3) * k.s4 + h * dqk;
  const int64_t voff = (int64_t)(kv_i3_zero ? 0 : kb % v.e3) * v.s3 + (int64_t)(kb / v.e3) * v.s4 + h * dv;
  int64_t krow[kFewKeysMax], vrow[kFewKeysMax];
#pragma unroll
  for (int j = 0; j < kFewKeysMax; ++j) {
    const int jj = j < Lk ? j : 0;
    krow[j] = koff + (int64_t)(jj % k.e1) * k.s1 + (int64_t)(jj / k.e1) * k.s2;
    vrow[j] = voff + (int64_t)(jj % v.e1) * v.s1 + (int64_t)(jj / v.e1) * v.s2;
  }
  float sc[kFewKeysMax];
#pragma unroll
  for (int j = 0; j < kFewKeysMax; ++j) sc[j] = 0.f;
#pragma unroll
  for (int c = 0; c < d; c += 8) {
    const uint4 qv = *reinterpret_cast<const uint4*>(qp + c);
    const __half2* qh = reinterpret_cast<const __half2*>(&qv);
    float2 qf[4];
#pragma unroll
    for (int t = 0; t < 4; ++t) qf[t] = __half22float2(qh[t]);
#pragma unroll
    for (int j = 0; j < kFewKeysMax; ++j) {
      if (j < Lk) {
        const uint4 kv = __ldg(reinterpret_cast<const uint4*>(k.base + krow[j] + c));
        const __half2* kh = reinterpret_cast<const __half2*>(&kv);
#pragma unroll
        for (int t = 0; t < 4; ++t) {
          const float2 kf = __half22float2(kh[t]);
          sc[j] = fmaf(qf[t].x, kf.x, fmaf(qf[t].y, kf.y, sc[j]));
        }
      }
    }
  }
  float m = -INFINITY;
#pragma unroll
  for (int j = 0; j < kFewKeysMax; ++j)
    if (j < Lk) m = fmaxf(m, sc[j]);
  float sum = 0.f;
#pragma unroll
  for (int j = 0; j < kFewKeysMax; ++j) {
    sc[j] = j < Lk ? exp2f((sc[j] - m) * scale_log2) : 0.f;
    sum += sc[j];
  }
  const float inv = out_scale / sum;
  __half* op = out + (int64_t)(l % q.e1) * os1 + (int64_t)(l / q.e1) * os2 + (int64_t)(qb % q.e3) * os3 +
               (int64_t)(qb / q.e3) * os4 + h * d;
#pragma unroll
  for (int c = 0; c < d; c += 8) {
    float acc[8];
#pragma unroll
    for (int t = 0; t < 8; ++t) acc[t] = 0.f;
#pragma unroll
    for (int j = 0; j < kFewKeysMax; ++j) {
      if (j < Lk) {
        const uint4 vv = __ldg(reinterpret_cast<const uint4*>(v.base + vrow[j] + c));
        const __half2* vh = reinterpret_cast<const __half2*>(&vv);
#pragma unroll
        for (int t = 0; t < 4; ++t) {
          const float2 vf = __half22float2(vh[t]);
          acc[2 * t] = fmaf(sc[j], vf.x, acc[2 * t]);
          acc[2 * t + 1] = fmaf(sc[j], vf.y, acc[2 * t + 1]);
        }
      }
    }
    uint4 o;
    __half2* oh = reinterpret_cast<__half2*>(&o);
    if (accumulate) {
      const uint4 old = *reinterpret_cast<const uint4*>(op + c);
      const __half2* ho = reinterpret_cast<const __half2*>(&old);
#pragma unroll
      for (int t = 0; t < 4; ++t) {
        const float2 f = __half22float2(ho[t]);
        oh[t] = __floats2half2_rn(fmaf(acc[2 * t], inv, f.x), fmaf(acc[2 * t + 1], inv, f.y));
      }
    } else {
#pragma unroll
      for (int t = 0; t < 4; ++t) oh[t] = __floats2half2_rn(acc[2 * t] * inv, acc[2 * t + 1] * inv);
    }
    *reinterpret_cast<uint4*>(op + c) = o;
  }
}

// ---------------------------------------------------------------------------------------------------------------
// Short-key attention (text cross-attention: 77 keys shared by the F frames of an image group).  A tensor-path CTA would live
// for two 64-key steps, so its set-up (barrier init, TMA round trips) would dominate.  Here the
// 77 keys/values of a (key batch, head) are staged once per block in shared memory (zero-padded to 80 rows) and each warp
// walks 16-row query tiles with mma.sync.m16n8k16: S (16 x 80) and P stay in registers, V^T fragments come from
// ldmatrix.trans.  HBM-bound (Q in, O out).
// ---------------------------------------------------------------------------------------------------------------
constexpr int kShortKeysPad = 80;
template <int D>
struct ShortCfg {
  static constexpr int kLdw = (D / 2 + 31) / 32 * 32 + 4;      // row stride in 32-bit words: == 4 (mod 32) -> 8 rows x 4 words tile the banks
  static constexpr int kLd = 2 * kLdw;                          // in halves
  static constexpr int kSmem = 2 * kShortKeysPad * kLd * 2;     // K and V
};

template <int D>
__global__ void __launch_bounds__(128)
attn_shortkeys_kernel(ViewDev q, ViewDev k, ViewDev v, __half* out, int64_t os1, int64_t os2, int64_t os3, int64_t os4, int dqk,
                      int dv, float scale_log2, int kv_div, int kv_i3_zero, int accumulate, float out_scale, int rows_per_block) {
  using Cfg = ShortCfg<D>;
  constexpr int LD = Cfg::kLd;
  extern __shared__ __align__(16) uint8_t smraw[];
  __half* sK = reinterpret_cast<__half*>(smraw);
  __half* sV = sK + kShortKeysPad * LD;
  const int Lq = q.e1 * q.e2, Lk = k.e1 * k.e2;
  const int h = blockIdx.y, qb = blockIdx.z;
  const int kb = qb / kv_div;
  const int64_t koff = (int64_t)(kv_i3_zero ? 0 : kb % k.e3) * k.s3 + (int64_t)(kb / k.e3) * k.s4 + h * dqk;
  const int64_t voff = (int64_t)(kv_i3_zero ? 0 : kb % v.e3) * v.s3 + (int64_t)(kb / v.e3) * v.s4 + h * dv;
  constexpr int VPR = D / 8;   // 16-byte vectors per row
  for (int i = threadIdx.x; i < kShortKeysPad * VPR; i += blockDim.x) {
    const int j = i / VPR, c = i % VPR;
    uint4 kv4 = make_uint4(0, 0, 0, 0), vv4 = make_uint4(0, 0, 0, 0);
    if (j < Lk) {
      kv4 = __ldg(reinterpret_cast<const uint4*>(k.base + koff + (int64_t)(j % k.e1) * k.s1 + (int64_t)(j / k.e1) * k.s2) + c);
      vv4 = __ldg(reinterpret_cast<const uint4*>(v.base + voff + (int64_t)(j % v.e1) * v.s1 + (int64_t)(j / v.e1) * v.s2) + c);
    }
    *reinterpret_cast<uint4*>(sK + j * LD + c * 8) = kv4;
    *reinterpret_cast<uint4*>(sV + j * LD + c * 8) = vv4;
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;
  const int row_begin = blockIdx.x * rows_per_block;
  const int row_end = min(row_begin + rows_per_block, Lq);
  const int64_t qbase = (int64_t)(qb % q.e3) * q.s3 + (int64_t)(qb / q.e3) * q.s4 + h * dqk;
  const int64_t obase = (int64_t)(qb % q.e3) * os3 + (int64_t)(qb / q.e3) * os4 + h * D;
  constexpr int KS = (D + 15) / 16;
  constexpr int NT = kShortKeysPad / 8;    // 10 key n-tiles
  for (int r0 = row_begin + warp * 16; r0 < row_end; r0 += 64) {
    const int l_lo = r0 + g, l_hi = r0 + g + 8;
    const bool ok_lo = l_lo < row_end, ok_hi = l_hi < row_end;
    const __half* q_lo = q.base + qbase + (int64_t)(l_lo % q.e1) * q.s1 + (int64_t)(l_lo / q.e1) * q.s2;
    const __half* q_hi = q.base + qbase + (int64_t)(l_hi % q.e1) * q.s1 + (int64_t)(l_hi / q.e1) * q.s2;
    float s[NT][4];
#pragma unroll
    for (int nt = 0; nt < NT; ++nt) { s[nt][0] = 0.f; s[nt][1] = 0.f; s[nt][2] = 0.f; s[nt][3] = 0.f; }
#pragma unroll
    for (int kk = 0; kk < KS; ++kk) {
      const int d0 = kk * 16 + 2 * t;
      const bool hi_half = (kk * 16 + 8) < D;       // second 8-column half of this k-step inside the head?
      uint32_t a[4];
      a[0] = ok_lo ? __ldg(reinterpret_cast<const uint32_t*>(q_lo + d0)) : 0u;
      a[1] = ok_hi ? __ldg(reinterpret_cast<const uint32_t*>(q_hi + d0)) : 0u;
      a[2] = (ok_lo && hi_half) ? __ldg(reinterpret_cast<const uint32_t*>(q_lo + d0 + 8)) : 0u;
      a[3] = (ok_hi && hi_half) ? __ldg(reinterpret_cast<const uint32_t*>(q_hi + d0 + 8)) : 0u;
#pragma unroll
      for (int nt = 0; nt < NT; ++nt) {
        const __half* kr = sK + (nt * 8 + g) * LD + d0;
        const uint32_t b0 = *reinterpret_cast<const uint32_t*>(kr);
        const uint32_t b1 = hi_half ? *reinterpret_cast<const uint32_t*>(kr + 8) : 0u;
        mma_16816(s[nt], a, b0, b1);
      }
    }
    // ---- softmax over the Lk valid keys (columns nt*8 + 2t, +1); rows g (c0,c1) and g+8 (c2,c3) live in a quad
    float mx_lo = -INFINITY, mx_hi = -INFINITY;
#pragma unroll
    for (int nt = 0; nt < NT; ++nt) {
      const int key = nt * 8 + 2 * t;
      if (key >= Lk) { s[nt][0] = -INFINITY; s[nt][2] = -INFINITY; }
      if (key + 1 >= Lk) { s[nt][1] = -INFINITY; s[nt][3] = -INFINITY; }
      mx_lo = fmaxf(mx_lo, fmaxf(s[nt][0], s[nt][1]));
      mx_hi = fmaxf(mx_hi, fmaxf(s[nt][2], s[nt][3]));
    }
#pragma unroll
    for (int o = 1; o <= 2; o <<= 1) {
      mx_lo = fmaxf(mx_lo, __shfl_xor_sync(0xffffffffu, mx_lo, o));
      mx_hi = fmaxf(mx_hi, __shfl_xor_sync(0xffffffffu, mx_hi, o));
    }
    const float nl = -mx_lo * scale_log2, nh = -mx_hi * scale_log2;
    float sum_lo = 0.f, sum_hi = 0.f;
#pragma unroll
    for (int nt = 0; nt < NT; ++nt) {
      s[nt][0] = ex2_approx(fmaf(s[nt][0], scale_log2, nl)); s[nt][1] = ex2_approx(fmaf(s[nt][1], scale_log2, nl));
      s[nt][2] = ex2_approx(fmaf(s[nt][2], scale_log2, nh)); s[nt][3] = ex2_approx(fmaf(s[nt][3], scale_log2, nh));
      sum_lo += s[nt][0] + s[nt][1];
      sum_hi += s[nt][2] + s[nt][3];
    }
#pragma unroll
    for (int o = 1; o <= 2; o <<= 1) {
      sum_lo += __shfl_xor_sync(0xffffffffu, sum_lo, o);
      sum_hi += __shfl_xor_sync(0xffffffffu, sum_hi, o);
    }
    const float inv_lo = 1.0f / sum_lo, inv_hi = 1.0f / sum_hi;
    // P (normalised, fp16) as A fragments of the 5 key k-steps
    uint32_t pa[NT / 2][4];
#pragma unroll
    for (int kk = 0; kk < NT / 2; ++kk) {
      pa[kk][0] = pack_f16x2(s[2 * kk][0] * inv_lo, s[2 * kk][1] * inv_lo);
      pa[kk][1] = pack_f16x2(s[2 * kk][2] * inv_hi, s[2 * kk][3] * inv_hi);
      pa[kk][2] = pack_f16x2(s[2 * kk + 1][0] * inv_lo, s[2 * kk + 1][1] * inv_lo);
      pa[kk][3] = pack_f16x2(s[2 * kk + 1][2] * inv_hi, s[2 * kk + 1][3] * inv_hi);
    }
    __half* o_lo = out + obase + (int64_t)(l_lo % q.e1) * os1 + (int64_t)(l_lo / q.e1) * os2;
    __half* o_hi = out + obase + (int64_t)(l_hi % q.e1) * os1 + (int64_t)(l_hi / q.e1) * os2;
#pragma unroll
    for (int nt = 0; nt < D / 8; ++nt) {
      float o[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
      for (int kk = 0; kk < NT / 2; ++kk) {
        const uint32_t addr = smem_u32(sV + (kk * 16 + (lane & 15)) * LD + nt * 8);
        uint32_t b0, b1;
        asm volatile("ldmatrix.sync.aligned.m8n8.x2.trans.shared.b16 {%0, %1}, [%2];" : "=r"(b0), "=r"(b1) : "r"(addr));
        mma_16816(o, pa[kk], b0, b1);
      }
      const int col = nt * 8 + 2 * t;
      if (ok_lo) {
        float x0 = o[0] * out_scale, x1 = o[1] * out_scale;
        if (accumulate) { const float2 f = __half22float2(*reinterpret_cast<const __half2*>(o_lo + col)); x0 += f.x; x1 += f.y; }
        *reinterpret_cast<uint32_t*>(o_lo + col) = pack_f16x2(x0, x1);
      }
      if (ok_hi) {
        float x0 = o[2] * out_scale, x1 = o[3] * out_scale;
        if (accumulate) { const float2 f = __half22float2(*reinterpret_cast<const __half2*>(o_hi + col)); x0 += f.x; x1 += f.y; }
        *reinterpret_cast<uint32_t*>(o_hi + col) = pack_f16x2(x0, x1);
      }
    }
  }
}

static ViewDev view_dev(const a3d_view5& v) {
  return ViewDev{reinterpret_cast<const __half*>(v.base), v.s1, v.s2, v.s3, v.s4, v.e1, v.e2, v.e3, v.e4};
}

static int tile_geom(const a3d_view5& v, int* box1, int* box2, int* t1, int* tiles, int* rows) {
  if (v.e1 >= 128) {
    // a ragged last tile reads rows past e1 as TMA's zero fill; with e2 > 1 they would be the next i2's rows instead
    if ((v.e1 % 128) && v.e2 != 1)
      return fail(A3D_EINVAL, "a3d_attention: inner extent %d is not a multiple of 128 and needs e2 == 1 (got %d)", v.e1, v.e2);
    *box1 = 128; *box2 = 1; *t1 = (v.e1 + 127) / 128; *tiles = *t1 * v.e2; *rows = 128;
  } else {
    int b2 = 128 / v.e1;
    if (b2 > v.e2) b2 = v.e2;
    if (b2 < 1 || v.e2 % b2) return fail(A3D_EINVAL, "a3d_attention: extents (%d,%d) do not tile", v.e1, v.e2);
    *box1 = v.e1; *box2 = b2; *t1 = 1; *tiles = v.e2 / b2; *rows = v.e1 * b2;
  }
  return 0;
}

static int view_map(const a3d_view5& v, int box1, int box2, const CUtensorMap** out) {
  const uint64_t dims[5] = {(uint64_t)v.cols, (uint64_t)v.e1, (uint64_t)v.e2, (uint64_t)v.e3, (uint64_t)v.e4};
  const uint64_t str[4] = {(uint64_t)v.s1, (uint64_t)v.s2, (uint64_t)v.s3, (uint64_t)v.s4};
  const uint32_t box[5] = {64, (uint32_t)box1, (uint32_t)box2, 1, 1};
  MapKey k = make_key(v.base, dims, str, box);
  return get_tensor_map(k, out);
}

// key tiles of 64 rows
static int tile_geom_k64(const a3d_view5& v, int* box1, int* box2, int* t1, int* tiles, int* rows_last) {
  if (v.e1 >= 64) {
    *box1 = 64; *box2 = 1; *t1 = (v.e1 + 63) / 64; *tiles = *t1 * v.e2;
    *rows_last = (v.e1 % 64) ? (v.e1 % 64) : 64;
    if ((v.e1 % 64) && v.e2 != 1) return fail(A3D_EINVAL, "a3d_attention: ragged key extent %d needs e2 == 1", v.e1);
  } else {
    int b2 = 64 / v.e1;
    if (b2 > v.e2) b2 = v.e2;
    if (b2 < 1 || v.e2 % b2) return fail(A3D_EINVAL, "a3d_attention: key extents (%d,%d) do not tile", v.e1, v.e2);
    *box1 = v.e1; *box2 = b2; *t1 = 1; *tiles = v.e2 / b2; *rows_last = v.e1 * b2;
  }
  return 0;
}

enum { kAttnFewKeys = 0, kAttnShortKeys = 1, kAttnTc = 2 };
static const char* const kAttnNames[] = {"fewkeys", "shortkeys", "tc"};   // indexed by kAttn*

// What one a3d_attention call launches, decided from its arguments alone: a3d_attention launches exactly this, and
// a3d_attention_kernel names it.
struct AttnPlan {
  int kernel;                         // kAttn*
  int dqk, dv, kv_div, batches;
  int qb1, qb2, qt1, qtiles, qrows;   // tensor-core kernel: 128-row query tiles (tile_geom)
  int kb1, kb2, kt1, ktiles, klast;   // ... and 64-row key tiles (tile_geom_k64)
};

static int plan_attention(const a3d_attn_args* a, AttnPlan* p) {
  if (!a || !a->q.base || !a->k.base || !a->v.base || !a->out) return fail(A3D_EINVAL, "a3d_attention: null operand");
  const int d = a->d;
  if (d != 40 && d != 80 && d != 160) return fail(A3D_EINVAL, "a3d_attention: head dim %d not in {40,80,160}", d);
  if (a->k.e1 != a->v.e1 || a->k.e2 != a->v.e2 || a->k.e3 != a->v.e3 || a->k.e4 != a->v.e4)
    return fail(A3D_EINVAL, "a3d_attention: K and V extents differ");
  memset(p, 0, sizeof(*p));
  p->dqk = (d + 15) / 16 * 16;
  p->dv = (d + 1 + 15) / 16 * 16;
  p->kv_div = a->kv_div > 0 ? a->kv_div : 1;
  const int batches = p->batches = a->q.e3 * a->q.e4;
  if ((batches + p->kv_div - 1) / p->kv_div > a->k.e3 * a->k.e4 && !a->kv_i3_zero)
    return fail(A3D_EINVAL, "a3d_attention: key batches (%d) do not cover query batches (%d / %d)", a->k.e3 * a->k.e4,
                batches, p->kv_div);
  // AUTO picks the kernel by key count; A3D_GEMM_TC forces the tensor-core kernel (tests use it to keep its ragged-key paths
  // covered)
  if (a->impl != A3D_GEMM_AUTO && a->impl != A3D_GEMM_TC)
    return fail(A3D_EINVAL, "a3d_attention: impl %d is not A3D_GEMM_AUTO or A3D_GEMM_TC", a->impl);
  if ((a->os1 | a->os2 | a->os3 | a->os4) % 8 || (reinterpret_cast<uintptr_t>(a->out) & 15))
    return fail(A3D_EINVAL, "a3d_attention: output rows must be 16-byte aligned");
  const bool auto_impl = a->impl == A3D_GEMM_AUTO;
  if (auto_impl && a->k.e1 * a->k.e2 <= kFewKeysMax) {
    // a handful of keys (IP-adapter image tokens): HBM-bound thread-per-(row, head) kernel, see attn_fewkeys_kernel
    if ((a->q.s1 | a->q.s2 | a->q.s3 | a->q.s4 | a->k.s1 | a->k.s2 | a->k.s3 | a->k.s4 | a->v.s1 | a->v.s2 | a->v.s3 | a->v.s4) % 8 ||
        ((reinterpret_cast<uintptr_t>(a->q.base) | reinterpret_cast<uintptr_t>(a->k.base) | reinterpret_cast<uintptr_t>(a->v.base)) & 15))
      return fail(A3D_EINVAL, "a3d_attention: operand rows must be 16-byte aligned");
    p->kernel = kAttnFewKeys;
    return A3D_OK;
  }
  if (auto_impl && a->k.e1 * a->k.e2 <= kShortKeysPad && (a->os1 | a->os2) % 2 == 0 &&
      ((a->k.s1 | a->k.s2 | a->k.s3 | a->k.s4 | a->v.s1 | a->v.s2 | a->v.s3 | a->v.s4) % 8 == 0) &&
      ((a->q.s1 | a->q.s2 | a->q.s3 | a->q.s4) % 2 == 0) &&
      ((reinterpret_cast<uintptr_t>(a->k.base) | reinterpret_cast<uintptr_t>(a->v.base)) & 15) == 0 &&
      (reinterpret_cast<uintptr_t>(a->q.base) & 3) == 0 && batches <= 65535) {
    // 9..80 keys (text cross-attention): warp-level MMA kernel with the keys resident in shared memory
    p->kernel = kAttnShortKeys;
    return A3D_OK;
  }
  p->kernel = kAttnTc;
  if (int r = tile_geom(a->q, &p->qb1, &p->qb2, &p->qt1, &p->qtiles, &p->qrows)) return r;
  if (batches > 65535 || a->heads > 65535) return fail(A3D_EINVAL, "a3d_attention: grid too large");
  return tile_geom_k64(a->k, &p->kb1, &p->kb2, &p->kt1, &p->ktiles, &p->klast);
}

template <int D>
static int launch_fewkeys(const a3d_attn_args* a, const AttnPlan& p, cudaStream_t st) {
  const int64_t total = (int64_t)p.batches * a->heads * a->q.e1 * a->q.e2;
  attn_fewkeys_kernel<D><<<(unsigned)((total + 255) / 256), 256, 0, st>>>(
      view_dev(a->q), view_dev(a->k), view_dev(a->v), reinterpret_cast<__half*>(a->out), a->os1, a->os2, a->os3, a->os4,
      a->heads, p.dqk, p.dv, a->scale * 1.4426950408889634f, p.kv_div, a->kv_i3_zero, a->accumulate, a->out_scale);
  A3D_LAUNCH_CHECK();
  return A3D_OK;
}

template <int D>
static int launch_shortkeys(const a3d_attn_args* a, const AttnPlan& p, cudaStream_t st) {
  using Cfg = ShortCfg<D>;
  static bool attr_set = false;
  if (!attr_set && Cfg::kSmem > 48 * 1024) {
    A3D_CUDA_CHECK(cudaFuncSetAttribute(attn_shortkeys_kernel<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmem));
    attr_set = true;
  }
  const int Lq = a->q.e1 * a->q.e2;
  int rows_per_block = 256;                       // 4 x 64-row rounds per block amortise the K/V staging
  while (rows_per_block > 64 && (int64_t)((Lq + rows_per_block - 1) / rows_per_block) * a->heads * p.batches < 8 * sm_count())
    rows_per_block /= 2;
  dim3 grid((unsigned)((Lq + rows_per_block - 1) / rows_per_block), (unsigned)a->heads, (unsigned)p.batches);
  attn_shortkeys_kernel<D><<<grid, 128, Cfg::kSmem, st>>>(view_dev(a->q), view_dev(a->k), view_dev(a->v),
                                                          reinterpret_cast<__half*>(a->out), a->os1, a->os2, a->os3, a->os4,
                                                          p.dqk, p.dv, a->scale * 1.4426950408889634f, p.kv_div, a->kv_i3_zero,
                                                          a->accumulate, a->out_scale, rows_per_block);
  A3D_LAUNCH_CHECK();
  return A3D_OK;
}

static unsigned long long* g_attn_dbg = nullptr;

template <int D>
static int launch_attn(const a3d_attn_args* a, const AttnPlan& p, cudaStream_t st) {
  using Cfg = AttnCfg<D>;
  AttnDev dev;
  memset(&dev, 0, sizeof(dev));
  dev.q_tiles = p.qtiles; dev.rows_q = p.qrows;
  dev.kv_tiles = p.ktiles; dev.rows_k = p.klast;
  dev.heads = a->heads;
  dev.q_t1 = p.qt1; dev.q_box1 = p.qb1; dev.q_box2 = p.qb2; dev.q_e1 = a->q.e1; dev.q_e3 = a->q.e3;
  dev.k_t1 = p.kt1; dev.k_box1 = p.kb1; dev.k_box2 = p.kb2; dev.k_e3 = a->k.e3;
  dev.kv_div = p.kv_div; dev.kv_i3_zero = a->kv_i3_zero;
  dev.q_box_bytes = 128u * p.qrows;
  dev.k_box_bytes = 128u * (uint32_t)(p.kb1 * p.kb2);
  dev.scale_log2 = a->scale * 1.4426950408889634f;
  dev.out = reinterpret_cast<__half*>(a->out);
  dev.os1 = a->os1; dev.os2 = a->os2; dev.os3 = a->os3; dev.os4 = a->os4;
  dev.accumulate = a->accumulate;
  dev.out_scale = a->out_scale;
  dev.dbg = g_attn_dbg;
  const CUtensorMap *mq, *mk, *mv;
  if (int r = view_map(a->q, p.qb1, p.qb2, &mq)) return r;
  if (int r = view_map(a->k, p.kb1, p.kb2, &mk)) return r;
  if (int r = view_map(a->v, p.kb1, p.kb2, &mv)) return r;
  static bool attr_set = false;
  if (!attr_set) {
    A3D_CUDA_CHECK(cudaFuncSetAttribute(attn_tc_kernel<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes));
    attr_set = true;
  }
  attn_tc_kernel<D><<<dim3(p.qtiles, a->heads, p.batches), kAttnThreads, Cfg::kSmemBytes, st>>>(dev, *mq, *mk, *mv);
  A3D_LAUNCH_CHECK();
  return A3D_OK;
}

template <int D>
static int launch_planned(const a3d_attn_args* a, const AttnPlan& p, cudaStream_t st) {
  switch (p.kernel) {
    case kAttnFewKeys: return launch_fewkeys<D>(a, p, st);
    case kAttnShortKeys: return launch_shortkeys<D>(a, p, st);
    default: return launch_attn<D>(a, p, st);
  }
}

}  // namespace a3d

extern "C" int a3d_attention_kernel(const a3d_attn_args* a, char* name, size_t n) {
  using namespace a3d;
  AttnPlan p;
  if (int r = plan_attention(a, &p)) return r;
  return kernel_name(name, n, "%s", kAttnNames[p.kernel]);
}

extern "C" int a3d_attention(const a3d_attn_args* a, void* stream) {
  using namespace a3d;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  AttnPlan p;
  if (int r = plan_attention(a, &p)) return r;
  switch (a->d) {
    case 40: return launch_planned<40>(a, p, st);
    case 80: return launch_planned<80>(a, p, st);
    default: return launch_planned<160>(a, p, st);
  }
}

// debug hook (not part of the product path): device counter the softmax of the tensor-core kernel bumps whenever a warp takes
// the lazy-rescale branch (tests assert that adversarial inputs really exercise it); null switches it off
extern "C" int a3d_debug_set_attn_trace(void* device_counter_u64) {
  a3d::g_attn_dbg = reinterpret_cast<unsigned long long*>(device_counter_u64);
  return A3D_OK;
}
