// a3d_gemm: C = epilogue(A * B^T) on Hopper tensor cores (wgmma).
//   * persistent, warp-specialised: warp 8 = TMA producer, warpgroups 0 and 1 = consumers; each consumer warpgroup owns 64 rows
//     of the 128-row tile, issues wgmma.mma_async on the staged operands and runs the epilogue straight from its fp32
//     accumulator registers while the producer already fills the ring for the next tile
//   * operands staged by TMA into 128B-swizzled shared memory (K-major) through a ring of mbarrier-guarded stages
//   * the tile's bias slice and the row-bias rows of a warpgroup's 64 rows are copied into that warpgroup's shared-memory
//     buffer (cp.async) under the tile's main loop, so the epilogue reads them without a global round trip
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
  int stages;     // operand ring depth
  int rb_slots;   // row-bias rows a warpgroup's buffer holds (gemm_rb_slots)
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

template <typename T>
__device__ __forceinline__ T perm_row(T m, T a, T b) {
  if (a == 0) return m;
  const T ab = a * b;
  return (m / ab) * ab + (m % b) * a + (m / b) % a;
}

constexpr int kBM = 128;
constexpr int kBK = 64;
constexpr int kGemmThreads = 288;   // 2 consumer warpgroups + 1 producer warp

constexpr int kGemmSmemMax = 227 * 1024;
constexpr int kMaxStages = 6;

// Shared memory: the operand ring (stages x kStageBytes, 1024-aligned), its barriers, then one epilogue buffer per consumer
// warpgroup: the tile's bias slice (row 0) and rb_slots row-bias rows, kEpiLd floats apart.  The epilogue reads 8 bytes per
// lane; with kEpiLd = 8 mod 32 the four row groups of a half-warp land on 32 distinct banks even when each reads its own row.
template <int BN>
struct GemmCfg {
  static constexpr int kABytes = kBM * kBK * 2;
  static constexpr int kBBytes = BN * kBK * 2;
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kEpiLd = BN + 8;
  static constexpr int epi_bytes(int rb_slots) { return 2 * (1 + rb_slots) * kEpiLd * 4; }
  // as many stages as fit next to the epilogue buffers, at most kMaxStages
  static constexpr int stages(int rb_slots) {
    return (kGemmSmemMax - 1024 - 256 - epi_bytes(rb_slots)) / kStageBytes > kMaxStages
               ? kMaxStages
               : (kGemmSmemMax - 1024 - 256 - epi_bytes(rb_slots)) / kStageBytes;
  }
  static constexpr int smem_bytes(int stages, int rb_slots) {
    return stages * kStageBytes + 1024 /*align slack*/ + 256 /*barriers*/ + epi_bytes(rb_slots);
  }
};
// a warpgroup's 64 rows use at most 64 row-bias rows; the 256-column tile falls back to 128 columns when they leave room for
// fewer than two stages (gemm_rb_slots)
static_assert(GemmCfg<128>::stages(64) >= 2 && GemmCfg<160>::stages(64) >= 2, "shared memory budget");
static_assert(GemmCfg<256>::stages(16) >= 3, "shared memory budget");

template <int BN>
__device__ __forceinline__ void wgmma_tile(float (&d)[BN / 2], uint64_t adesc, uint64_t bdesc, uint32_t acc) {
  if constexpr (BN == 256) wgmma_ss_n256<0>(d, adesc, bdesc, acc);
  else if constexpr (BN == 160) wgmma_ss_n160<0>(d, adesc, bdesc, acc);
  else wgmma_ss_n128<0>(d, adesc, bdesc, acc);
}

// EPI: 0 = bias/row-bias only, 1 = + residuals / row permutation, 2 = GEGLU, 3 = fp32 output, 4 = GELU of the biased value
enum { kEpiPlain = 0, kEpiRes = 1, kEpiGeglu = 2, kEpiF32 = 3, kEpiGelu = 4 };

// The epilogue walks a thread's 8-column groups in chunks of G groups, both of its rows at once.  Bias and row-bias come
// from the warpgroup's shared-memory buffer; the only global operands are the residuals (kEpiRes).  Those of a chunk are
// requested together, and those of the next chunk before the current one is stored, so a thread waits for memory once per
// chunk rather than once per group and row.  A GEGLU chunk holds G / 2 value groups and their gates.  The residuals sit in
// registers next to the accumulators, and a 288-thread CTA puts three warps on one SM sub-partition, which caps a thread at
// 168 registers.  At BN = 256 the 128 accumulator registers leave room for one group's residuals only, so there the next
// group is requested after the current one is stored.  Residual rows are fetched into L2 ahead of the epilogue (see the
// main loop).
template <int BN, int EPI>
struct EpiChunk {
  static constexpr int G = BN == 256 && EPI == kEpiRes ? 1 : 2;
  static constexpr bool kAhead = G == 2;
  uint32_t r1[2][G], r2[2][G];        // [row][group] fp16x2 residuals (kEpiRes only)
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

// 4-byte copies: the ABI guarantees bias / row-bias 4-byte alignment only
__device__ __forceinline__ void cp_async_4(uint32_t smem_dst, const void* src) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(smem_dst), "l"(src) : "memory");
}
// ordered with the epilogue's global stores like the global loads it replaces: a plain load would be hoisted over them,
// and the loads of every chunk would then compete with the accumulators for registers
__device__ __forceinline__ float2 lds_f32x2(uint32_t a) {
  float2 v;
  asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "r"(a) : "memory");
  return v;
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }
// barrier of one consumer warpgroup (ids 1, 2; 0 is __syncthreads)
__device__ __forceinline__ void warpgroup_sync(int wg) {
  if (wg == 0) asm volatile("bar.sync 1, 128;" ::: "memory");
  else asm volatile("bar.sync 2, 128;" ::: "memory");
}

template <int BN, int EPI>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_tc_kernel(const GemmDev p, const __grid_constant__ CUtensorMap mapA, const __grid_constant__ CUtensorMap mapB) {
  static_assert(EPI != kEpiGeglu || BN % 64 == 0, "GEGLU pairs a value with its gate inside 64-column blocks");
  static_assert((BN / 8) % EpiChunk<BN, EPI>::G == 0, "the tile's column groups split into whole chunks");
  using Cfg = GemmCfg<BN>;
  const int num_stages = p.stages;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + num_stages * Cfg::kABytes;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + num_stages * Cfg::kStageBytes);   // [num_stages]
  uint64_t* empty_bar = full_bar + num_stages;                                              // [num_stages]
  float* epi_buf = reinterpret_cast<float*>(smem + num_stages * Cfg::kStageBytes + 256);    // [2][1 + rb_slots][kEpiLd]

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int num_tiles = p.tiles_m * p.tiles_n;

  if (warp == 8 && lane == 0) {
    tma_prefetch_desc(&mapA);
    tma_prefetch_desc(&mapB);
    for (int i = 0; i < num_stages; ++i) {
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
          if (++stage == num_stages) { stage = 0; phase ^= 1; }
        }
      }
    }
    return;
  }

  // -------------------------------------------------------------------- consumers: 2 warpgroups x 64 rows
  const int wg = warp >> 2;
  const int g = lane >> 2, t = lane & 3;
  const uint32_t epi = smem_u32(epi_buf + wg * (1 + p.rb_slots) * Cfg::kEpiLd);
  int stage = 0;
  uint32_t phase = 0;
  float acc[BN / 2];
  // one loop counter (tcount); the tile index is derived from it rather than kept live across the main loop
  for (int tcount = 0; (int)(blockIdx.x + tcount * gridDim.x) < num_tiles; ++tcount) {
    const int tile = blockIdx.x + tcount * gridDim.x;
    const int mt = tile / p.tiles_n, nt = tile % p.tiles_n;
    const bool tr = p.trace && blockIdx.x == 0 && threadIdx.x == 0 && tcount < 60;
    if (tr) p.trace[tcount * 16 + 0] = clock64();
    // epilogue rows of this thread: row[h] = 16 w + g + 8 h of the warpgroup's 64; group j = columns 8 j + 2 t, +1.
    // R2 and C are read / written at the same (orow, n) by the same thread, so R2 may be C.  R1 is read at (row, n), which
    // another thread writes when the rows are permuted: R1 must not alias C then (see a3d.h).  Row indices are divided in
    // 32 bits (a3d_gemm checks that they fit): a 64-bit division is a subroutine call, and with the 128 accumulator
    // registers of BN = 256 live, ptxas spills around it.
    const int col_base = nt * BN + 2 * t;
    uint32_t row[2], orow[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      row[h] = (uint32_t)mt * kBM + wg * 64 + (warp & 3) * 16 + g + 8 * h;
      orow[h] = (EPI == kEpiRes) ? perm_row<uint32_t>(row[h], (uint32_t)p.perm_a, (uint32_t)p.perm_b) : row[h];
    }
    // ---- epilogue buffer, filled under the main loop once every thread of the warpgroup is done with the previous tile's.
    // Row-bias rows m0 .. m1 (those < M) of the warpgroup use table rows q % rb_mod, q = q0 .. m1 / rb_div; slot s holds
    // table row (q0 + s) % rb_mod and row m reads slot (m / rb_div - q0) % nslots: when the window wraps (nslots = rb_mod)
    // the modulo keeps the slots distinct.  Columns past N are zero-filled, not read.  Bits 16 h .. 16 h + 15 of rb_off:
    // the float offset in epi of this thread's columns 2 t, 2 t + 1 of row h's slot, 0xffff without a row-bias or past M
    // (one register: it stays live across the main loop next to the accumulators).
    uint32_t rb_off = 0xffffffffu;
    {
      const int64_t n0 = (int64_t)nt * BN;
      const int ncols = p.N - n0 < BN ? (int)(p.N - n0) : BN;
      const uint32_t m0 = (uint32_t)mt * kBM + wg * 64, M = (uint32_t)p.M;
      const uint32_t rb_div = (uint32_t)p.rb_div, rb_mod = (uint32_t)p.rb_mod;
      uint32_t nslots = 0, q = 0;
      if (p.rowbias && m0 < M) {
        const uint32_t m1 = m0 + 63 < M ? m0 + 63 : M - 1;
        const uint32_t q0 = m0 / rb_div;
        nslots = m1 / rb_div - q0 + 1 < rb_mod ? m1 / rb_div - q0 + 1 : rb_mod;
#pragma unroll
        for (int h = 0; h < 2; ++h)
          if (row[h] < M)
            rb_off ^= (0xffffu ^ ((1 + (row[h] / rb_div - q0) % nslots) * Cfg::kEpiLd + 2 * t)) << 16 * h;
        q = q0 % rb_mod;
      }
      if (tcount > 0) warpgroup_sync(wg);
      for (uint32_t r = p.bias ? 0 : 1; r <= nslots; ++r) {
        const float* src = (r == 0 ? p.bias : p.rowbias + q * p.rb_ld) + n0;
        const uint32_t dst = epi + 4 * r * Cfg::kEpiLd;
        for (int c = threadIdx.x & 127; c < BN; c += 128) {
          if (c < ncols) cp_async_4(dst + 4 * c, src + c);
          else asm volatile("st.shared.f32 [%0], %1;" ::"r"(dst + 4 * c), "f"(0.f) : "memory");
        }
        if (r > 0 && ++q == rb_mod) q = 0;
      }
    }
    // ---- main loop: one wgmma group in flight; the stage of k-block kb-1 is released once group kb-1 has retired
    int prev_stage = -1;
    for (int kb = 0; kb < p.num_k_blocks; ++kb) {
      if constexpr (EPI == kEpiRes) {
        // the residual rows of this tile into L2 two k-blocks before the epilogue reads them: far enough ahead to cover an
        // HBM miss, close enough that the operand stream of a long-K tile does not evict them first.  The four lanes of a
        // row take its 128-byte lines t, t + 4 (a row's BN halves span at most 2 BN / 128 + 1 lines).
        if (kb == (p.num_k_blocks > 2 ? p.num_k_blocks - 2 : 0)) {
          const int ncols = p.N - nt * BN < BN ? (int)p.N - nt * BN : BN;
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
            fetch(p.R1 + row[h] * p.ldr1 + nt * BN, p.R1 && row[h] < p.M);
            fetch(p.R2 + orow[h] * p.ldr2 + nt * BN, p.R2 && row[h] < p.M);
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
      if (++stage == num_stages) { stage = 0; phase ^= 1; }
    }

    // ---- epilogue from registers, chunk by chunk (EpiChunk): chunk c covers groups epi_group(c, 0 .. G - 1) of both rows
    using Chunk = EpiChunk<BN, EPI>;
    constexpr int G = Chunk::G;
    constexpr int kChunks = BN / 8 / G;
    Chunk op;
    auto load_chunk = [&](int c) {
      if constexpr (EPI == kEpiRes) {
#pragma unroll
        for (int s = 0; s < G; ++s) {
          const int64_t n = col_base + 8 * epi_group<EPI, G>(c, s);
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const bool ok = n < p.N && row[h] < p.M;
            // coherent loads, unlike __ldg: they cannot be hoisted above the previous chunk's stores, which would hold the
            // operands of every chunk in registers at once
            op.r1[h][s] = (p.R1 && ok) ? *reinterpret_cast<const uint32_t*>(p.R1 + row[h] * p.ldr1 + n) : 0u;
            op.r2[h][s] = (p.R2 && ok) ? *reinterpret_cast<const uint32_t*>(p.R2 + orow[h] * p.ldr2 + n) : 0u;
          }
        }
      }
    };
    // same order as the SIMT kernel: (acc + bias + row-bias) * acc_scale, then + r1_scale R1, + R2; columns 8 j + 2 t, +1
    // of row h
    auto finish = [&](float v0, float v1, int h, int j) {
      if (p.bias) {
        const float2 b = lds_f32x2(epi + 4 * (2 * t + 8 * j));
        v0 += b.x; v1 += b.y;
      }
      const uint32_t off = (rb_off >> 16 * h) & 0xffffu;
      if (off != 0xffffu) {
        const float2 r = lds_f32x2(epi + 4 * (off + 8 * j));
        v0 += r.x; v1 += r.y;
      }
      return make_float2(v0 * p.acc_scale, v1 * p.acc_scale);
    };
    auto half2_float2 = [](uint32_t u) { return __half22float2(*reinterpret_cast<const __half2*>(&u)); };

    if constexpr (Chunk::kAhead) load_chunk(0);   // under the last MMA group
    cp_async_wait_all();
    warpgroup_sync(wg);
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
            const float2 u = finish(acc[4 * ju + 2 * h], acc[4 * ju + 2 * h + 1], h, ju);
            const float2 gt = finish(acc[4 * jg + 2 * h], acc[4 * jg + 2 * h + 1], h, jg);
            out[h][s] = pack_f16x2(u.x * gelu_erf(gt.x), u.y * gelu_erf(gt.y));
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
        float2 out[2][G];
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int s = 0; s < G; ++s) {
            const int j = c * G + s;
            out[h][s] = finish(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1], h, j);
          }
        if (Chunk::kAhead && c + 1 < kChunks) load_chunk(c + 1);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          if (row[h] >= p.M) continue;
          float* crow = reinterpret_cast<float*>(p.C) + row[h] * p.ldc;
#pragma unroll
          for (int s = 0; s < G; ++s) {
            const int64_t n = col_base + 8 * (c * G + s);
            if (n >= p.N) continue;
            crow[n] = out[h][s].x;
            crow[n + 1] = out[h][s].y;
          }
        }
      } else {
        uint32_t out[2][G];
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int s = 0; s < G; ++s) {
            const int j = c * G + s;
            const float2 f = finish(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1], h, j);
            float v0 = f.x, v1 = f.y;
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

// Row-bias rows the 64 rows of one warpgroup use: their quotients m / rb_div span at most ceil(63 / rb_div) + 1 values,
// and at most rb_mod of them are distinct table rows (rb_mod is at most the number of quotients of all M rows, see plan_gemm).
static int gemm_rb_slots(const GemmDev& d) {
  if (!d.rowbias) return 0;
  const int64_t s = 63 / d.rb_div + (63 % d.rb_div != 0) + 1;
  return (int)(d.rb_mod < s ? d.rb_mod : s);
}

// GemmCfg<BN> at a run-time tile width
static int gemm_stages(int bn, int rb_slots) {
  return bn == 256 ? GemmCfg<256>::stages(rb_slots) : bn == 160 ? GemmCfg<160>::stages(rb_slots) : GemmCfg<128>::stages(rb_slots);
}
static int gemm_smem_bytes(int bn, int stages, int rb_slots) {
  return bn == 256   ? GemmCfg<256>::smem_bytes(stages, rb_slots)
         : bn == 160 ? GemmCfg<160>::smem_bytes(stages, rb_slots)
                     : GemmCfg<128>::smem_bytes(stages, rb_slots);
}

// What one a3d_gemm call launches, decided from its arguments alone: a3d_gemm launches exactly this, and a3d_gemm_kernel
// names it.
struct GemmPlan {
  GemmDev dev;        // the kernel's arguments (trace excepted)
  SimtConv cv;        // CONV3 geometry (SIMT kernel and the A tensor map)
  bool simt;
  int bn, epi;        // tensor-core tile width and epilogue instance (kEpi*)
  int smem;           // dynamic shared memory of the tensor-core kernel
  const char* geom;   // A operand tiling: plain, conv-wide-rows, conv-row-block or conv-image-block
};

static const char* const kEpiNames[] = {"plain", "res", "geglu", "f32", "gelu"};   // indexed by kEpi*

static int plan_gemm(const a3d_gemm_args* a, GemmPlan* p) {
  if (!a || !a->A || !a->B || !a->C) return fail(A3D_EINVAL, "a3d_gemm: null operand");
  if (a->M <= 0 || a->N <= 0 || a->K <= 0) return fail(A3D_EINVAL, "a3d_gemm: empty problem M=%lld N=%lld K=%lld",
                                                        (long long)a->M, (long long)a->N, (long long)a->K);
  memset(p, 0, sizeof(*p));
  GemmDev& d = p->dev;
  d.M = a->M; d.N = a->N; d.K = a->K;
  d.a_mode = a->a_mode;
  d.bias = a->bias; d.rowbias = a->rowbias; d.rb_ld = a->rb_ld;
  d.rb_div = a->rb_div > 0 ? a->rb_div : 1; d.rb_mod = a->rb_mod > 0 ? a->rb_mod : (int64_t)1 << 40;
  // rows m < M only: a divisor above M leaves every quotient 0, and a modulus above the largest quotient changes none, so
  // both are clamped to M's range (the tensor-core kernel divides in 32 bits)
  if (d.rb_div > d.M) d.rb_div = d.M;
  if (d.rb_mod > (d.M - 1) / d.rb_div + 1) d.rb_mod = (d.M - 1) / d.rb_div + 1;
  d.acc_scale = a->acc_scale;   // the caller passes 1.0 when unused; 0 is a legitimate blend weight, not a sentinel
  d.R1 = reinterpret_cast<const __half*>(a->R1); d.ldr1 = a->ldr1; d.r1_scale = a->r1_scale;
  d.R2 = reinterpret_cast<const __half*>(a->R2); d.ldr2 = a->ldr2;
  d.C = a->C; d.ldc = a->ldc; d.geglu = a->geglu; d.out_f32 = a->out_f32;
  d.perm_a = a->perm_a; d.perm_b = a->perm_b;
  if (a->geglu < 0 || a->geglu > 2) return fail(A3D_EINVAL, "a3d_gemm: geglu must be 0 (none), 1 (GEGLU) or 2 (GELU)");
  const bool geglu = a->geglu == 1;
  if (geglu && (a->out_f32 || a->R1 || a->R2 || a->perm_a || (a->N % 128)))
    return fail(A3D_EINVAL, "a3d_gemm: GEGLU epilogue takes bias / row-bias only, fp16 output, N %% 128 == 0");
  if (a->geglu == 2 && (a->out_f32 || a->R1 || a->R2 || a->perm_a))
    return fail(A3D_EINVAL, "a3d_gemm: GELU epilogue takes bias / row-bias only, fp16 output");
  if (a->out_f32 && (a->R1 || a->R2 || a->perm_a))
    return fail(A3D_EINVAL, "a3d_gemm: fp32 output supports bias / row-bias only");
  if (a->impl != A3D_GEMM_AUTO && a->impl != A3D_GEMM_TC && a->impl != A3D_GEMM_SIMT)
    return fail(A3D_EINVAL, "a3d_gemm: impl %d is not A3D_GEMM_AUTO, _TC or _SIMT", a->impl);

  SimtConv& cv = p->cv;
  cv = SimtConv{0, 0, 0, 0, 1, 0, 0};
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
  // the kernel's row and column indices (up to M + 127, N + 255) and the permutation period perm_a * perm_b are 32-bit
  tc_ok = tc_ok && a->M <= INT32_MAX - kBM && a->N <= INT32_MAX - 256 &&
          (a->perm_a == 0 || (a->perm_a <= INT32_MAX && a->perm_b <= INT32_MAX / a->perm_a));
  p->geom = "plain";
  d.bimg = 1; d.tpr = 1;
  if (a->a_mode == A3D_A_CONV3) {
    tc_ok = tc_ok && (cv.c % kBK == 0);
    const int opix = cv.oh * cv.ow;
    if (cv.ow > kBM) {           // wide images (VAE at 256^2): a tile is a 128-pixel piece of one output row
      tc_ok = tc_ok && (cv.ow % kBM == 0);
      d.boh = 1; d.tpr = cv.ow / kBM; d.tpi = cv.oh * d.tpr;
      p->geom = "conv-wide-rows";
    } else if (opix >= kBM) {
      tc_ok = tc_ok && (opix % kBM == 0) && (kBM % cv.ow == 0);
      d.boh = kBM / cv.ow; d.tpi = opix / kBM;
      p->geom = "conv-row-block";
    } else {
      tc_ok = tc_ok && (kBM % opix == 0);
      d.boh = cv.oh; d.bimg = kBM / (opix > 0 ? opix : 1);
      p->geom = "conv-image-block";
    }
    tc_ok = tc_ok && (d.tpr > 1 ? kBM : cv.ow) * cv.s <= 256 && d.boh * cv.s <= 256;
    d.cpb = cv.c / kBK;
    d.conv_pad = cv.pad;
  }
  if (a->R1) tc_ok = tc_ok && (a->ldr1 % 16 == 0) && ((reinterpret_cast<uintptr_t>(a->R1) & 31) == 0);
  if (a->R2) tc_ok = tc_ok && (a->ldr2 % 16 == 0) && ((reinterpret_cast<uintptr_t>(a->R2) & 31) == 0);
  if (a->impl == A3D_GEMM_TC && !tc_ok)
    return fail(A3D_EINVAL, "a3d_gemm: shape/alignment not supported by the tensor-core path (M=%lld N=%lld K=%lld)",
                (long long)a->M, (long long)a->N, (long long)a->K);
  if (a->impl == A3D_GEMM_SIMT || !tc_ok) {
    p->simt = true;
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
  d.rb_slots = gemm_rb_slots(d);
  // a table with up to 64 distinct rows per warpgroup (CLIP's position embeddings) leaves room for fewer than two stages
  // of the 256-column tile
  if (BN == 256 && GemmCfg<256>::stages(d.rb_slots) < 2) BN = 128;
  d.stages = gemm_stages(BN, d.rb_slots);
  p->smem = gemm_smem_bytes(BN, d.stages, d.rb_slots);
  if (d.stages < 2 || p->smem > kGemmSmemMax)
    return fail(A3D_EINVAL, "a3d_gemm: %d row-bias rows per warpgroup leave no room for the operand ring", d.rb_slots);
  if (geglu && a->N % BN) return fail(A3D_EINVAL, "a3d_gemm: GEGLU needs N %% 128 == 0");
  d.num_k_blocks = (int)(a->K / kBK);
  d.tiles_m = (int)((a->M + kBM - 1) / kBM);
  d.tiles_n = (int)((a->N + BN - 1) / BN);
  p->bn = BN;
  p->epi = a->out_f32 ? kEpiF32 : geglu ? kEpiGeglu : a->geglu == 2 ? kEpiGelu : (a->R1 || a->R2 || a->perm_a) ? kEpiRes : kEpiPlain;
  return A3D_OK;
}

template <int BN, int EPI>
static int launch_tc_epi(const GemmPlan& p, const CUtensorMap* mapA, const CUtensorMap* mapB, cudaStream_t st) {
  static bool attr_set = false;
  if (!attr_set) {
    A3D_CUDA_CHECK(cudaFuncSetAttribute(gemm_tc_kernel<BN, EPI>, cudaFuncAttributeMaxDynamicSharedMemorySize, kGemmSmemMax));
    attr_set = true;
  }
  const int tiles = p.dev.tiles_m * p.dev.tiles_n;
  const int grid = tiles < sm_count() ? tiles : sm_count();
  gemm_tc_kernel<BN, EPI><<<grid, kGemmThreads, p.smem, st>>>(p.dev, *mapA, *mapB);
  A3D_LAUNCH_CHECK();
  return A3D_OK;
}

template <int BN>
static int launch_tc(const GemmPlan& p, const CUtensorMap* mapA, const CUtensorMap* mapB, cudaStream_t st) {
  switch (p.epi) {
    case kEpiF32: return launch_tc_epi<BN, kEpiF32>(p, mapA, mapB, st);
    case kEpiGeglu:
      if constexpr (BN % 64 == 0) return launch_tc_epi<BN, kEpiGeglu>(p, mapA, mapB, st);
      else return fail(A3D_EINVAL, "a3d_gemm: GEGLU needs a 128- or 256-column tile");
    case kEpiGelu: return launch_tc_epi<BN, kEpiGelu>(p, mapA, mapB, st);
    case kEpiRes: return launch_tc_epi<BN, kEpiRes>(p, mapA, mapB, st);
    default: return launch_tc_epi<BN, kEpiPlain>(p, mapA, mapB, st);
  }
}

static long long* g_gemm_trace = nullptr;

}  // namespace a3d

// debug hook (not part of the product path): per-tile clock64 timestamps of CTA 0 of the following tensor-core GEMM launches
extern "C" int a3d_debug_set_gemm_trace(void* device_buffer_1024_int64) {
  a3d::g_gemm_trace = reinterpret_cast<long long*>(device_buffer_1024_int64);
  return A3D_OK;
}

extern "C" int a3d_gemm_kernel(const a3d_gemm_args* a, char* name, size_t n) {
  using namespace a3d;
  GemmPlan p;
  if (int r = plan_gemm(a, &p)) return r;
  if (p.simt) return kernel_name(name, n, "simt");
  return kernel_name(name, n, "tc BN%d %s %s", p.bn, kEpiNames[p.epi], p.geom);
}

extern "C" int a3d_gemm(const a3d_gemm_args* a, void* stream) {
  using namespace a3d;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  GemmPlan p;
  if (int r = plan_gemm(a, &p)) return r;
  p.dev.trace = g_gemm_trace;
  const SimtConv& cv = p.cv;
  if (p.simt) {
    const int64_t n_out = a->geglu == 1 ? a->N / 2 : a->N;
    const int64_t total = a->M * n_out;
    const int threads = 128;
    const int64_t blocks = (total + threads - 1) / threads;
    gemm_simt_kernel<<<(unsigned)blocks, threads, 0, st>>>(p.dev, reinterpret_cast<const __half*>(a->A), a->lda,
                                                           reinterpret_cast<const __half*>(a->B), cv);
    A3D_LAUNCH_CHECK();
    return A3D_OK;
  }

  const CUtensorMap *mapA = nullptr, *mapB = nullptr;
  {
    const uint64_t dims[5] = {(uint64_t)a->K, (uint64_t)a->N, 1, 1, 1};
    const uint64_t str[4] = {(uint64_t)a->K, (uint64_t)a->K * a->N, (uint64_t)a->K * a->N, (uint64_t)a->K * a->N};
    const uint32_t box[5] = {kBK, (uint32_t)p.bn, 1, 1, 1};
    MapKey kb = make_key(a->B, dims, str, box);
    if (int r = get_tensor_map(kb, &mapB)) return r;
  }
  if (a->a_mode == A3D_A_PLAIN) {
    const uint64_t dims[5] = {(uint64_t)a->K, (uint64_t)a->M, 1, 1, 1};
    const uint64_t str[4] = {(uint64_t)a->lda, (uint64_t)a->lda * a->M, (uint64_t)a->lda * a->M, (uint64_t)a->lda * a->M};
    const uint32_t box[5] = {kBK, kBM, 1, 1, 1};
    MapKey ka = make_key(a->A, dims, str, box);
    if (int r = get_tensor_map(ka, &mapA)) return r;
  } else {
    const GemmDev& d = p.dev;
    const uint64_t img = (uint64_t)cv.h * cv.w * cv.c;
    const uint64_t dims[5] = {(uint64_t)cv.c, (uint64_t)cv.w, (uint64_t)cv.h, (uint64_t)cv.n, 1};
    const uint64_t str[4] = {(uint64_t)cv.c, (uint64_t)cv.w * cv.c, img, img * cv.n};
    const uint32_t box[5] = {kBK, (uint32_t)((d.tpr > 1 ? kBM : cv.ow) * cv.s), (uint32_t)(d.boh * cv.s), (uint32_t)d.bimg, 1};
    MapKey ka = make_key(a->A, dims, str, box);
    ka.estr[1] = cv.s; ka.estr[2] = cv.s;
    if (int r = get_tensor_map(ka, &mapA)) return r;
  }
  switch (p.bn) {
    case 256: return launch_tc<256>(p, mapA, mapB, st);
    case 160: return launch_tc<160>(p, mapA, mapB, st);
    default: return launch_tc<128>(p, mapA, mapB, st);
  }
}
