// a3d_gemm: C = epilogue(A * B^T) on Hopper tensor cores (wgmma).
//   * persistent, warp-specialised: warp 8 = TMA producer, warpgroups 0 and 1 = consumers; each consumer warpgroup owns 64 rows
//     of the 128-row tile, issues wgmma.mma_async on the staged operands and runs the epilogue straight from its fp32
//     accumulator registers while the producer already fills the ring for the next tile
//   * operands staged by TMA into 128B-swizzled shared memory (K-major) through a ring of mbarrier-guarded stages
//   * A3D_A_CONV3: the A operand is an implicit 3x3 im2col of an NHWC image -- each k-block is one (tap, 64-channel)
//     slice fetched with a rank-4 TMA box whose out-of-bounds rows/cols are zero-filled by the hardware (= padding 1);
//     stride-2 convolutions use the tensor map's traversal strides
// Replaces torch linear/conv2d (cuBLAS/cuDNN) under the diffusers blocks driven by
// animatediff/models/unet_motion_mv_model.py:768-859 of the reference.
#include <type_traits>

#include "a3d_common.cuh"
#include "a3d_host.cuh"
#include "a3d_wgmma.cuh"

namespace a3d {

struct GemmDev {
  int64_t M, N, K;
  int num_k_blocks;
  int tiles_m, tiles_n;
  // conv A addressing
  int a_mode;
  int cpb;        // 64-channel blocks per tap (C/64)
  int conv_s;     // stride
  int tpi;        // output tiles per image (>=1) or 0 when several images share a tile
  int boh;        // output rows per tile
  int bimg;       // images per tile
  int tpr;        // tiles per output row (> 1 when an output row is wider than the 128-row tile)
  int conv_pad;   // zero padding in front of row / column 0 (1, or 0 for the asymmetric (0,1,0,1) padding of the VAE downsampler)
  // epilogue
  const float* bias;
  const float* rowbias;
  int64_t rb_ld, rb_div, rb_mod;
  float acc_scale;
  const __half* R1; int64_t ldr1; float r1_scale;
  const __half* R2; int64_t ldr2;
  void* C; int64_t ldc;
  int geglu, out_f32;
  int64_t perm_a, perm_b;
  long long* trace;   // debug: per-tile clock64 timestamps of CTA 0 (null in production), see a3d_debug_set_gemm_trace
};

// gelu(x) = 0.5 x (1 + erf(x / sqrt 2)) with erf from Abramowitz-Stegun 7.1.26 (|err| <= 1.5e-7, far below fp16 output
// resolution): 1 rcp + 1 ex2 on the XU pipe + 11 FMA-pipe instructions instead of erff's ~30 (the GEGLU epilogue is ALU-bound)
__device__ __forceinline__ float gelu_erf(float x) {
  // gelu(x) = x/2 + |x|/2 erf(|x| / sqrt 2);  erf(z) = 1 - (a1 t + .. + a5 t^5) exp(-z^2), t = 1 / (1 + 0.3275911 z).  Constants folded so
  // that one evaluation is 7 FFMA + 4 FMUL + MUFU.RCP + MUFU.EX2
  float t;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t) : "f"(fmaf(0.3275911f * 0.70710678118654752f, fabsf(x), 1.0f)));
  float poly = fmaf(1.061405429f, t, -1.453152027f);
  poly = fmaf(poly, t, 1.421413741f);
  poly = fmaf(poly, t, -0.284496736f);
  poly = fmaf(poly, t, 0.254829592f);
  const float xs = x * 0.84932180028801904f;              // sqrt(log2(e) / 2): exp(-x^2 / 2) = 2^(-xs^2)
  const float e = ex2_approx(-xs * xs);
  const float erf_abs = fmaf(-(poly * t), e, 1.0f);
  const float h = 0.5f * x;
  return fmaf(fabsf(h), erf_abs, h);
}

__device__ __forceinline__ int64_t perm_row(int64_t m, int64_t a, int64_t b) {
  if (a == 0) return m;
  const int64_t ab = a * b;
  return (m / ab) * ab + (m % b) * a + (m / b) % a;
}

constexpr int kBM = 128;
constexpr int kBK = 64;
constexpr int kGemmThreads = 288;   // 2 consumer warpgroups + 1 producer warp

template <int BN>
struct GemmCfg {
  static constexpr int kABytes = kBM * kBK * 2;
  static constexpr int kBBytes = BN * kBK * 2;
  static constexpr int kStageBytes = kABytes + kBBytes;
  // as many stages as fit next to nothing else: the epilogue works from registers and needs no shared memory
  static constexpr int kStages = (227 * 1024 - 1024 - 256) / kStageBytes > 6 ? 6 : (227 * 1024 - 1024 - 256) / kStageBytes;
  static constexpr int kSmemBytes = kStages * kStageBytes + 1024 /*align slack*/ + 256 /*barriers*/;
  static_assert(kSmemBytes <= 227 * 1024, "shared memory budget");
};

template <int BN>
__device__ __forceinline__ void wgmma_tile(float (&d)[BN / 2], uint64_t adesc, uint64_t bdesc, uint32_t acc) {
  if constexpr (BN == 256) wgmma_ss_n256<0>(d, adesc, bdesc, acc);
  else if constexpr (BN == 160) wgmma_ss_n160<0>(d, adesc, bdesc, acc);
  else wgmma_ss_n128<0>(d, adesc, bdesc, acc);
}

// EPI: 0 = bias/row-bias only, 1 = + residuals / row permutation, 2 = GEGLU, 3 = fp32 output, 4 = GELU of the biased value
enum { kEpiPlain = 0, kEpiRes = 1, kEpiGeglu = 2, kEpiF32 = 3, kEpiGelu = 4 };

// The epilogue walks a thread's 8-column groups in chunks of G groups, both of its rows at once.  All global operands of a
// chunk are requested together, and (kAhead) those of the next chunk before the current one is stored, so a thread waits for
// memory once per chunk rather than once per group and row.  A GEGLU chunk holds G / 2 value groups and their gates.  The
// operands sit in registers next to the accumulators, and a 288-thread CTA puts three warps on one SM sub-partition, which
// caps a thread at 168 registers.  At BN = 256 the 128 accumulator registers leave room for one chunk's operands only, so
// there the next chunk is requested after the current one is stored.  Residual rows are fetched into L2 ahead of the
// epilogue at every BN (see the main loop).
template <int BN, int EPI>
struct EpiChunk {
  static constexpr int G = BN == 256 ? 1 + (EPI == kEpiGeglu) : 2;
  static constexpr bool kAhead = BN != 256;
  float bias[G][2];
  float rb[2][G][2];                  // [row][group][column]
  uint32_t r1[2][G], r2[2][G];        // fp16x2 residuals (kEpiRes only)
};

// accumulator group (8 columns) of slot s of chunk c; GEGLU: slots < G / 2 hold values u of output group o, the others
// their gates, 4 groups further (the accumulator columns come as (u[32] | g[32]) blocks)
template <int EPI, int G>
__device__ __forceinline__ constexpr int epi_group(int c, int s) {
  if constexpr (EPI != kEpiGeglu) {
    return c * G + s;
  } else {
    const int o = c * (G / 2) + s % (G / 2);
    return (o / 4) * 8 + o % 4 + (s >= G / 2 ? 4 : 0);
  }
}

__device__ __forceinline__ void prefetch_l2(const void* a) { asm volatile("prefetch.global.L2 [%0];" ::"l"(a)); }

template <int BN, int EPI>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_tc_kernel(const GemmDev p, const __grid_constant__ CUtensorMap mapA, const __grid_constant__ CUtensorMap mapB) {
  static_assert(EPI != kEpiGeglu || BN % 64 == 0, "GEGLU pairs a value with its gate inside 64-column blocks");
  static_assert((BN / 8) % EpiChunk<BN, EPI>::G == 0, "the tile's column groups split into whole chunks");
  using Cfg = GemmCfg<BN>;
  constexpr int kStages = Cfg::kStages;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + kStages * Cfg::kABytes;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + kStages * Cfg::kStageBytes);   // [kStages]
  uint64_t* empty_bar = full_bar + kStages;                                              // [kStages]

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int num_tiles = p.tiles_m * p.tiles_n;

  if (warp == 8 && lane == 0) {
    tma_prefetch_desc(&mapA);
    tma_prefetch_desc(&mapB);
    for (int i = 0; i < kStages; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 8);   // one arrive per consumer warp
    }
    mbar_fence_init();
  }
  __syncthreads();

  if (warp == 8) {
    // ------------------------------------------------------------------ TMA producer (one thread)
    if (lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int mt = tile / p.tiles_n, nt = tile % p.tiles_n;
        int img0 = 0, oh0 = 0, ow0 = 0;
        if (p.a_mode == A3D_A_CONV3) {
          if (p.tpr > 1) { img0 = mt / p.tpi; oh0 = (mt % p.tpi) / p.tpr; ow0 = ((mt % p.tpi) % p.tpr) * kBM; }
          else if (p.tpi > 0) { img0 = mt / p.tpi; oh0 = (mt % p.tpi) * p.boh; }
          else { img0 = mt * p.bimg; oh0 = 0; }
        }
        for (int kb = 0; kb < p.num_k_blocks; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1);
          mbar_expect_tx(&full_bar[stage], Cfg::kStageBytes);
          if (p.a_mode == A3D_A_CONV3) {
            const int tap = kb / p.cpb, c0 = (kb % p.cpb) * kBK;
            const int ky = tap / 3, kx = tap % 3;
            tma_load_5d(smem_a + stage * Cfg::kABytes, &mapA, &full_bar[stage], c0, ow0 * p.conv_s + kx - p.conv_pad,
                        oh0 * p.conv_s + ky - p.conv_pad, img0, 0);
          } else {
            tma_load_5d(smem_a + stage * Cfg::kABytes, &mapA, &full_bar[stage], kb * kBK, mt * kBM, 0, 0, 0);
          }
          tma_load_5d(smem_b + stage * Cfg::kBBytes, &mapB, &full_bar[stage], kb * kBK, nt * BN, 0, 0, 0);
          if (++stage == kStages) { stage = 0; phase ^= 1; }
        }
      }
    }
    return;
  }

  // -------------------------------------------------------------------- consumers: 2 warpgroups x 64 rows
  const int wg = warp >> 2;
  const int g = lane >> 2, t = lane & 3;
  int stage = 0;
  uint32_t phase = 0;
  int tcount = 0;
  float acc[BN / 2];
  for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x, ++tcount) {
    const int mt = tile / p.tiles_n, nt = tile % p.tiles_n;
    const bool tr = p.trace && blockIdx.x == 0 && threadIdx.x == 0 && tcount < 60;
    if (tr) p.trace[tcount * 16 + 0] = clock64();
    // epilogue rows of this thread: row[h] = 16 w + g + 8 h of the warpgroup's 64; group j = columns 8 j + 2 t, +1.
    // R2 and C are read / written at the same (orow, n) by the same thread, so R2 may be C.  R1 is read at (row, n), which
    // another thread writes when the rows are permuted: R1 must not alias C then (see a3d.h).
    const int64_t col_base = (int64_t)nt * BN + 2 * t;
    int64_t row[2], orow[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      row[h] = (int64_t)mt * kBM + wg * 64 + (warp & 3) * 16 + g + 8 * h;
      orow[h] = (EPI == kEpiRes) ? perm_row(row[h], p.perm_a, p.perm_b) : row[h];
    }
    // ---- main loop: one wgmma group in flight; the stage of k-block kb-1 is released once group kb-1 has retired
    int prev_stage = -1;
    for (int kb = 0; kb < p.num_k_blocks; ++kb) {
      if constexpr (EPI == kEpiRes) {
        // the residual rows of this tile into L2 two k-blocks before the epilogue reads them: far enough ahead to cover an
        // HBM miss, close enough that the operand stream of a long-K tile does not evict them first.  The four lanes of a
        // row take its 128-byte lines t, t + 4 (a row's BN halves span at most 2 BN / 128 + 1 lines).
        if (kb == (p.num_k_blocks > 2 ? p.num_k_blocks - 2 : 0)) {
          const int64_t ncols = p.N - (int64_t)nt * BN < BN ? p.N - (int64_t)nt * BN : BN;
          auto fetch = [&](const __half* a, bool ok) {
            const uintptr_t e = reinterpret_cast<uintptr_t>(a + ncols), l0 = reinterpret_cast<uintptr_t>(a) & ~uintptr_t(127);
#pragma unroll
            for (int i = 0; i < (2 * BN / 128 + 4) / 4; ++i) {
              const uintptr_t l = l0 + 128 * (t + 4 * i);
              if (ok && l < e) prefetch_l2(reinterpret_cast<const void*>(l));
            }
          };
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            fetch(p.R1 + row[h] * p.ldr1 + (int64_t)nt * BN, p.R1 && row[h] < p.M);
            fetch(p.R2 + orow[h] * p.ldr2 + (int64_t)nt * BN, p.R2 && row[h] < p.M);
          }
        }
      }
      mbar_wait(&full_bar[stage], phase);
      const uint32_t a0 = smem_u32(smem_a + stage * Cfg::kABytes + wg * (64 * 128));
      const uint32_t b0 = smem_u32(smem_b + stage * Cfg::kBBytes);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < kBK / 16; ++k)
        wgmma_tile<BN>(acc, make_smem_desc_sw128(a0 + 32 * k, 16, 1024), make_smem_desc_sw128(b0 + 32 * k, 16, 1024),
                       (kb | k) ? 1u : 0u);
      wgmma_commit();
      wgmma_wait<1>();
      if (prev_stage >= 0 && lane == 0) mbar_arrive(&empty_bar[prev_stage]);
      prev_stage = stage;
      if (++stage == kStages) { stage = 0; phase ^= 1; }
    }

    // ---- epilogue from registers, chunk by chunk (EpiChunk): chunk c covers groups epi_group(c, 0 .. G - 1) of both rows
    using Chunk = EpiChunk<BN, EPI>;
    constexpr int G = Chunk::G;
    constexpr int kChunks = BN / 8 / G;
    const float* rb[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) rb[h] = p.rowbias ? p.rowbias + ((row[h] / p.rb_div) % p.rb_mod) * p.rb_ld : nullptr;
    Chunk op;
    auto load_chunk = [&](int c) {
#pragma unroll
      for (int s = 0; s < G; ++s) {
        const int64_t n = col_base + 8 * epi_group<EPI, G>(c, s);
        const bool col_ok = n < p.N;
        // coherent loads, unlike __ldg: they cannot be hoisted above the previous chunk's stores, which would hold the
        // operands of every chunk in registers at once
        op.bias[s][0] = (p.bias && col_ok) ? p.bias[n] : 0.f;
        op.bias[s][1] = (p.bias && col_ok) ? p.bias[n + 1] : 0.f;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const bool ok = col_ok && row[h] < p.M;
          op.rb[h][s][0] = (rb[h] && ok) ? rb[h][n] : 0.f;
          op.rb[h][s][1] = (rb[h] && ok) ? rb[h][n + 1] : 0.f;
          if constexpr (EPI == kEpiRes) {
            op.r1[h][s] = (p.R1 && ok) ? *reinterpret_cast<const uint32_t*>(p.R1 + row[h] * p.ldr1 + n) : 0u;
            op.r2[h][s] = (p.R2 && ok) ? *reinterpret_cast<const uint32_t*>(p.R2 + orow[h] * p.ldr2 + n) : 0u;
          }
        }
      }
    };
    // same order as the SIMT kernel: (acc + bias + row-bias) * acc_scale, then + r1_scale R1, + R2
    auto finish = [&](float v, int h, int s, int e) {
      if (p.bias) v += op.bias[s][e];
      if (rb[h]) v += op.rb[h][s][e];
      return v * p.acc_scale;
    };
    auto half2_float2 = [](uint32_t u) { return __half22float2(*reinterpret_cast<const __half2*>(&u)); };

    if constexpr (Chunk::kAhead) load_chunk(0);   // under the last MMA group
    wgmma_wait<0>();
    reg_fence(acc);
    if (lane == 0) mbar_arrive(&empty_bar[prev_stage]);
    if (tr) p.trace[tcount * 16 + 1] = clock64();

#pragma unroll
    for (int c = 0; c < kChunks; ++c) {
      if constexpr (!Chunk::kAhead) load_chunk(c);
      if constexpr (EPI == kEpiGeglu) {
        uint32_t out[2][G / 2];
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int s = 0; s < G / 2; ++s) {
            const int ju = epi_group<EPI, G>(c, s), jg = epi_group<EPI, G>(c, s + G / 2);
            const float u0 = finish(acc[4 * ju + 2 * h], h, s, 0), u1 = finish(acc[4 * ju + 2 * h + 1], h, s, 1);
            const float g0 = finish(acc[4 * jg + 2 * h], h, s + G / 2, 0), g1 = finish(acc[4 * jg + 2 * h + 1], h, s + G / 2, 1);
            out[h][s] = pack_f16x2(u0 * gelu_erf(g0), u1 * gelu_erf(g1));
          }
        if (Chunk::kAhead && c + 1 < kChunks) load_chunk(c + 1);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          if (row[h] >= p.M) continue;
          __half* crow = reinterpret_cast<__half*>(p.C) + row[h] * p.ldc;
#pragma unroll
          for (int s = 0; s < G / 2; ++s) {
            if (col_base + 8 * epi_group<EPI, G>(c, s) >= p.N) continue;
            const int o = c * (G / 2) + s;   // output group: columns 8 o + 2 t, +1 of the tile's BN / 2
            *reinterpret_cast<uint32_t*>(crow + (int64_t)nt * (BN / 2) + 8 * o + 2 * t) = out[h][s];
          }
        }
      } else if constexpr (EPI == kEpiF32) {
        float out[2][G][2];
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int s = 0; s < G; ++s)
#pragma unroll
            for (int e = 0; e < 2; ++e) out[h][s][e] = finish(acc[4 * (c * G + s) + 2 * h + e], h, s, e);
        if (Chunk::kAhead && c + 1 < kChunks) load_chunk(c + 1);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          if (row[h] >= p.M) continue;
          float* crow = reinterpret_cast<float*>(p.C) + row[h] * p.ldc;
#pragma unroll
          for (int s = 0; s < G; ++s) {
            const int64_t n = col_base + 8 * (c * G + s);
            if (n >= p.N) continue;
            crow[n] = out[h][s][0];
            crow[n + 1] = out[h][s][1];
          }
        }
      } else {
        uint32_t out[2][G];
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int s = 0; s < G; ++s) {
            const int j = c * G + s;
            float v0 = finish(acc[4 * j + 2 * h], h, s, 0), v1 = finish(acc[4 * j + 2 * h + 1], h, s, 1);
            if constexpr (EPI == kEpiGelu) {
              v0 = gelu_erf(v0); v1 = gelu_erf(v1);
            }
            if constexpr (EPI == kEpiRes) {
              if (p.R1) {
                const float2 f = half2_float2(op.r1[h][s]);
                v0 += p.r1_scale * f.x; v1 += p.r1_scale * f.y;
              }
              if (p.R2) {
                const float2 f = half2_float2(op.r2[h][s]);
                v0 += f.x; v1 += f.y;
              }
            }
            out[h][s] = pack_f16x2(v0, v1);
          }
        if (Chunk::kAhead && c + 1 < kChunks) load_chunk(c + 1);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          if (row[h] >= p.M) continue;
          __half* crow = reinterpret_cast<__half*>(p.C) + orow[h] * p.ldc;
#pragma unroll
          for (int s = 0; s < G; ++s) {
            const int64_t n = col_base + 8 * (c * G + s);
            if (n >= p.N) continue;
            *reinterpret_cast<uint32_t*>(crow + n) = out[h][s];
          }
        }
      }
    }
    if (tr) p.trace[tcount * 16 + 2] = clock64();
  }
}

// ---------------------------------------------------------------------------------------------------------------
// SIMT bring-up / reference kernel: same semantics, one thread per output element (also serves odd shapes)
// ---------------------------------------------------------------------------------------------------------------
struct SimtConv { int n, h, w, c, s, oh, ow, pad; };

__global__ void gemm_simt_kernel(const GemmDev p, const __half* __restrict__ A, int64_t lda, const __half* __restrict__ B,
                                 SimtConv cv) {
  const int64_t n_out = p.geglu == 1 ? p.N / 2 : p.N;
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= p.M * n_out) return;
  const int64_t m = idx / n_out;
  const int64_t j = idx % n_out;
  auto dot = [&](int64_t n) {
    float acc = 0.f;
    const __half* b = B + n * p.K;
    if (p.a_mode == A3D_A_PLAIN) {
      const __half* a = A + m * lda;
      for (int64_t k = 0; k < p.K; ++k) acc += __half2float(a[k]) * __half2float(b[k]);
    } else {
      const int img = (int)(m / (cv.oh * cv.ow));
      const int oy = (int)((m / cv.ow) % cv.oh), ox = (int)(m % cv.ow);
      for (int tap = 0; tap < 9; ++tap) {
        const int iy = oy * cv.s + tap / 3 - cv.pad, ix = ox * cv.s + tap % 3 - cv.pad;
        if (iy < 0 || iy >= cv.h || ix < 0 || ix >= cv.w) continue;
        const __half* a = A + (((int64_t)img * cv.h + iy) * cv.w + ix) * cv.c;
        const __half* bb = b + (int64_t)tap * cv.c;
        for (int c = 0; c < cv.c; ++c) acc += __half2float(a[c]) * __half2float(bb[c]);
      }
    }
    return acc;
  };
  const int64_t orow = perm_row(m, p.perm_a, p.perm_b);
  const float* rb = p.rowbias ? p.rowbias + ((m / p.rb_div) % p.rb_mod) * p.rb_ld : nullptr;
  auto finish = [&](int64_t n) {   // same epilogue order as the tensor-core kernel's finish()
    float v = dot(n);
    if (p.bias) v += p.bias[n];
    if (rb) v += rb[n];
    return v * p.acc_scale;
  };
  if (p.geglu == 1) {
    const int64_t blk = j / 32, e = j % 32;
    const int64_t nu = blk * 64 + e, ng = nu + 32;
    const float u = finish(nu), g = finish(ng);
    reinterpret_cast<__half*>(p.C)[orow * p.ldc + j] = __float2half_rn(u * gelu_erf(g));
    return;
  }
  float v = finish(j);
  if (p.geglu == 2) v = gelu_erf(v);
  if (p.R1) v += p.r1_scale * __half2float(p.R1[m * p.ldr1 + j]);
  if (p.R2) v += __half2float(p.R2[orow * p.ldr2 + j]);
  if (p.out_f32) reinterpret_cast<float*>(p.C)[orow * p.ldc + j] = v;
  else reinterpret_cast<__half*>(p.C)[orow * p.ldc + j] = __float2half_rn(v);
}

template <int BN, int EPI>
static int launch_tc_epi(const GemmDev& dev, const CUtensorMap* mapA, const CUtensorMap* mapB, cudaStream_t st) {
  using Cfg = GemmCfg<BN>;
  static bool attr_set = false;
  if (!attr_set) {
    A3D_CUDA_CHECK(cudaFuncSetAttribute(gemm_tc_kernel<BN, EPI>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmemBytes));
    attr_set = true;
  }
  const int tiles = dev.tiles_m * dev.tiles_n;
  const int grid = tiles < sm_count() ? tiles : sm_count();
  gemm_tc_kernel<BN, EPI><<<grid, kGemmThreads, Cfg::kSmemBytes, st>>>(dev, *mapA, *mapB);
  A3D_LAUNCH_CHECK();
  return A3D_OK;
}

template <int BN>
static int launch_tc(const GemmDev& dev, const CUtensorMap* mapA, const CUtensorMap* mapB, cudaStream_t st) {
  if (dev.out_f32) return launch_tc_epi<BN, kEpiF32>(dev, mapA, mapB, st);
  if (dev.geglu == 1) {
    if constexpr (BN % 64 == 0) return launch_tc_epi<BN, kEpiGeglu>(dev, mapA, mapB, st);
    else return fail(A3D_EINVAL, "a3d_gemm: GEGLU needs a 128- or 256-column tile");
  }
  if (dev.geglu == 2) return launch_tc_epi<BN, kEpiGelu>(dev, mapA, mapB, st);
  if (dev.R1 || dev.R2 || dev.perm_a) return launch_tc_epi<BN, kEpiRes>(dev, mapA, mapB, st);
  return launch_tc_epi<BN, kEpiPlain>(dev, mapA, mapB, st);
}

static long long* g_gemm_trace = nullptr;

}  // namespace a3d

// debug hook (not part of the product path): per-tile clock64 timestamps of CTA 0 of the following tensor-core GEMM launches
extern "C" int a3d_debug_set_gemm_trace(void* device_buffer_1024_int64) {
  a3d::g_gemm_trace = reinterpret_cast<long long*>(device_buffer_1024_int64);
  return A3D_OK;
}

extern "C" int a3d_gemm(const a3d_gemm_args* a, void* stream) {
  using namespace a3d;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (!a || !a->A || !a->B || !a->C) return fail(A3D_EINVAL, "a3d_gemm: null operand");
  if (a->M <= 0 || a->N <= 0 || a->K <= 0) return fail(A3D_EINVAL, "a3d_gemm: empty problem M=%lld N=%lld K=%lld",
                                                        (long long)a->M, (long long)a->N, (long long)a->K);
  GemmDev d;
  memset(&d, 0, sizeof(d));
  d.M = a->M; d.N = a->N; d.K = a->K;
  d.a_mode = a->a_mode;
  d.bias = a->bias; d.rowbias = a->rowbias; d.rb_ld = a->rb_ld;
  d.rb_div = a->rb_div > 0 ? a->rb_div : 1; d.rb_mod = a->rb_mod > 0 ? a->rb_mod : (int64_t)1 << 40;
  d.acc_scale = a->acc_scale;   // the caller passes 1.0 when unused; 0 is a legitimate blend weight, not a sentinel
  d.R1 = reinterpret_cast<const __half*>(a->R1); d.ldr1 = a->ldr1; d.r1_scale = a->r1_scale;
  d.R2 = reinterpret_cast<const __half*>(a->R2); d.ldr2 = a->ldr2;
  d.C = a->C; d.ldc = a->ldc; d.geglu = a->geglu; d.out_f32 = a->out_f32;
  d.perm_a = a->perm_a; d.perm_b = a->perm_b;
  d.trace = g_gemm_trace;
  if (a->geglu < 0 || a->geglu > 2) return fail(A3D_EINVAL, "a3d_gemm: geglu must be 0 (none), 1 (GEGLU) or 2 (GELU)");
  const bool geglu = a->geglu == 1;
  if (geglu && (a->out_f32 || a->R1 || a->R2 || a->perm_a || (a->N % 128)))
    return fail(A3D_EINVAL, "a3d_gemm: GEGLU epilogue takes bias / row-bias only, fp16 output, N %% 128 == 0");
  if (a->geglu == 2 && (a->out_f32 || a->R1 || a->R2 || a->perm_a))
    return fail(A3D_EINVAL, "a3d_gemm: GELU epilogue takes bias / row-bias only, fp16 output");
  if (a->out_f32 && (a->R1 || a->R2 || a->perm_a))
    return fail(A3D_EINVAL, "a3d_gemm: fp32 output supports bias / row-bias only");

  SimtConv cv{0, 0, 0, 0, 1, 0, 0};
  if (a->a_mode == A3D_A_CONV3) {
    const int s = a->conv_stride;
    if (s != 1 && s != 2) return fail(A3D_EINVAL, "a3d_gemm: conv stride must be 1 or 2");
    if (a->conv_h % s || a->conv_w % s) return fail(A3D_EINVAL, "a3d_gemm: conv H/W must be multiples of the stride");
    cv = SimtConv{a->conv_n, a->conv_h, a->conv_w, a->conv_c, s, a->conv_h / s, a->conv_w / s, a->conv_nopad_lo ? 0 : 1};
    if (a->K != 9LL * a->conv_c || a->M != (int64_t)cv.n * cv.oh * cv.ow)
      return fail(A3D_EINVAL, "a3d_gemm: conv geometry does not match M/K");
    d.conv_s = s;
  } else if (a->a_mode != A3D_A_PLAIN) {
    return fail(A3D_EINVAL, "a3d_gemm: unknown a_mode %d", a->a_mode);
  }

  // ---- can the tensor-core path take it?
  bool tc_ok = (a->K % kBK == 0) && (a->N % (geglu ? 16 : 8) == 0) && ((reinterpret_cast<uintptr_t>(a->A) & 15) == 0) &&
               ((reinterpret_cast<uintptr_t>(a->B) & 15) == 0) && (a->ldc % 16 == 0) &&
               ((reinterpret_cast<uintptr_t>(a->C) & 31) == 0);
  if (a->a_mode == A3D_A_PLAIN) tc_ok = tc_ok && (a->lda % 8 == 0) && a->lda >= a->K;
  int boh = 0, bimg = 1, tpi = 0, tpr = 1;
  if (a->a_mode == A3D_A_CONV3) {
    tc_ok = tc_ok && (cv.c % kBK == 0);
    const int opix = cv.oh * cv.ow;
    if (cv.ow > kBM) {           // wide images (VAE at 256^2): a tile is a 128-pixel piece of one output row
      tc_ok = tc_ok && (cv.ow % kBM == 0);
      boh = 1; tpr = cv.ow / kBM; tpi = cv.oh * tpr; bimg = 1;
    } else if (opix >= kBM) {
      tc_ok = tc_ok && (opix % kBM == 0) && (kBM % cv.ow == 0);
      boh = kBM / cv.ow; tpi = opix / kBM; bimg = 1;
    } else {
      tc_ok = tc_ok && (kBM % opix == 0);
      boh = cv.oh; tpi = 0; bimg = kBM / (opix > 0 ? opix : 1);
    }
    tc_ok = tc_ok && (tpr > 1 ? kBM : cv.ow) * cv.s <= 256 && boh * cv.s <= 256;
  }
  if (a->R1) tc_ok = tc_ok && (a->ldr1 % 16 == 0) && ((reinterpret_cast<uintptr_t>(a->R1) & 31) == 0);
  if (a->R2) tc_ok = tc_ok && (a->ldr2 % 16 == 0) && ((reinterpret_cast<uintptr_t>(a->R2) & 31) == 0);
  int impl = a->impl;
  if (impl == A3D_GEMM_AUTO) impl = tc_ok ? A3D_GEMM_TCGEN05 : A3D_GEMM_SIMT;
  if (impl == A3D_GEMM_TCGEN05 && !tc_ok)
    return fail(A3D_EINVAL, "a3d_gemm: shape/alignment not supported by the tensor-core path (M=%lld N=%lld K=%lld)",
                (long long)a->M, (long long)a->N, (long long)a->K);

  if (impl == A3D_GEMM_SIMT) {
    const int64_t n_out = geglu ? a->N / 2 : a->N;
    const int64_t total = a->M * n_out;
    const int threads = 128;
    const int64_t blocks = (total + threads - 1) / threads;
    gemm_simt_kernel<<<(unsigned)blocks, threads, 0, st>>>(d, reinterpret_cast<const __half*>(a->A), a->lda,
                                                           reinterpret_cast<const __half*>(a->B), cv);
    A3D_LAUNCH_CHECK();
    return A3D_OK;
  }

  // ---- tile shape
  int BN;
  if (geglu) BN = (a->N % 256 == 0) ? 256 : 128;
  else if (a->N % 256 == 0) BN = 256;
  else if (a->K <= 640 && a->N > 512 && (256 * ((a->N + 255) / 256) - a->N) * 8 <= a->N) {
    // short-K GEMMs are bound by the epilogue / output stores, where the 256-wide tile amortises the per-tile handshakes
    // best: a ragged last tile (<= 12.5% idle MMA columns) costs nothing there
    BN = 256;
  } else if (a->N % 160 == 0) BN = 160;
  else BN = 128;
  {
    static int force = -1;
    if (force < 0) { const char* e = getenv("A3D_GEMM_BN"); force = e ? atoi(e) : 0; }
    if (!geglu && (force == 128 || force == 160 || force == 256)) BN = force;   // tuning override
  }
  if (geglu && a->N % BN) return fail(A3D_EINVAL, "a3d_gemm: GEGLU needs N %% 128 == 0");
  d.num_k_blocks = (int)(a->K / kBK);
  d.tiles_m = (int)((a->M + kBM - 1) / kBM);
  d.tiles_n = (int)((a->N + BN - 1) / BN);
  d.cpb = a->a_mode == A3D_A_CONV3 ? cv.c / kBK : 0;
  d.tpi = tpi; d.boh = boh; d.bimg = bimg; d.tpr = tpr; d.conv_pad = cv.pad;
  const CUtensorMap *mapA = nullptr, *mapB = nullptr;
  {
    MapKey kb;
    const uint64_t dims[5] = {(uint64_t)a->K, (uint64_t)a->N, 1, 1, 1};
    const uint64_t str[4] = {(uint64_t)a->K, (uint64_t)a->K * a->N, (uint64_t)a->K * a->N, (uint64_t)a->K * a->N};
    const uint32_t box[5] = {kBK, (uint32_t)BN, 1, 1, 1};
    kb = make_key(a->B, dims, str, box);
    if (int r = get_tensor_map(kb, &mapB)) return r;
  }
  if (a->a_mode == A3D_A_PLAIN) {
    const uint64_t dims[5] = {(uint64_t)a->K, (uint64_t)a->M, 1, 1, 1};
    const uint64_t str[4] = {(uint64_t)a->lda, (uint64_t)a->lda * a->M, (uint64_t)a->lda * a->M, (uint64_t)a->lda * a->M};
    const uint32_t box[5] = {kBK, kBM, 1, 1, 1};
    MapKey ka = make_key(a->A, dims, str, box);
    if (int r = get_tensor_map(ka, &mapA)) return r;
  } else {
    const uint64_t img = (uint64_t)cv.h * cv.w * cv.c;
    const uint64_t dims[5] = {(uint64_t)cv.c, (uint64_t)cv.w, (uint64_t)cv.h, (uint64_t)cv.n, 1};
    const uint64_t str[4] = {(uint64_t)cv.c, (uint64_t)cv.w * cv.c, img, img * cv.n};
    const uint32_t box[5] = {kBK, (uint32_t)((tpr > 1 ? kBM : cv.ow) * cv.s), (uint32_t)(boh * cv.s), (uint32_t)bimg, 1};
    MapKey ka = make_key(a->A, dims, str, box);
    ka.estr[1] = cv.s; ka.estr[2] = cv.s;
    if (int r = get_tensor_map(ka, &mapA)) return r;
  }
  switch (BN) {
    case 256: return launch_tc<256>(d, mapA, mapB, st);
    case 160: return launch_tc<160>(d, mapA, mapB, st);
    default: return launch_tc<128>(d, mapA, mapB, st);
  }
}
