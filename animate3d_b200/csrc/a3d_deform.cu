// Per-frame deformation field of the 4D gaussians, all frames of a batch in one launch:
//   k-planes (HexPlane) lookup -- 2 scales x 6 planes, bilinear, border clamp, align_corners -- product over planes, concat
//   over scales -> 32 features -> three bias-free MLPs 32 -> 32 (ReLU) -> {3, 4, 3} -> xyz + d, exp(s + d), normalize(q + d)
// forward and backward (gradients to the plane grids and MLP weights; the static gaussians are frozen buffers in
// Animate3D, gaussian_4d.py:262-297).  The `use_global_trans` branch (gaussian_4d.py:499-511, 525-539) needs the MEAN feature
// vector of a frame before any output can be formed: kMode 2 computes those means (one extra pass over the L2-resident
// planes), the host evaluates the two 32-wide global MLPs + Euler matrix on [T, 32], and the main pass takes the rotated
// base quaternions as `rot_base`; backward returns d/d rot_base and folds d/d mean-feature back into the plane gradients.  Replaces, per (frame, gaussian), the 12 grid_sample + 6 GEMM + elementwise launches the
// reference issues PER CAMERA (custom/threestudio-animate3d/geometry/gaussian_4d.py:39-64, 450-548;
// renderer/diff_gaussian_rasterizer_advanced_4d.py:77-83, 119-135) and de-duplicates the 4 views of a frame.
#include "a3d_host.cuh"

namespace a3d {

constexpr int kPlanes = 6;
constexpr int kMaxScales = 2;
constexpr int kFeat = 16;                  // channels per plane
constexpr int kHid = 32;                   // MLP width == feature width (2 scales x 16)

struct DeformGrids {
  const float* plane[kMaxScales][kPlanes]; // [C, H, W]
  float* gplane[kMaxScales][kPlanes];      // gradients (backward) or null
  int h[kMaxScales][kPlanes], w[kMaxScales][kPlanes];
  int scales;
};

struct DeformMlp {          // row-major [out, in]
  const float *w1[3], *w2[3];              // 0: xyz (3), 1: rot (4), 2: scale (3)
  float *gw1[3], *gw2[3];
};

__device__ __constant__ int c_comb[kPlanes][2] = {{0, 1}, {0, 2}, {0, 3}, {1, 2}, {1, 3}, {2, 3}};
__device__ __forceinline__ int out_dim(int m) { return m == 1 ? 4 : 3; }

struct Bilerp {
  int x0, x1, y0, y1;
  float wx, wy;
};
// grid_sample(align_corners=True, padding_mode="border") coordinates for normalised (gx, gy): gx indexes W, gy indexes H
__device__ __forceinline__ Bilerp bilerp_setup(float gx, float gy, int W, int H) {
  float fx = (gx + 1.f) * 0.5f * (float)(W - 1);
  float fy = (gy + 1.f) * 0.5f * (float)(H - 1);
  fx = fminf(fmaxf(fx, 0.f), (float)(W - 1));
  fy = fminf(fmaxf(fy, 0.f), (float)(H - 1));
  Bilerp b;
  b.x0 = (int)floorf(fx); b.y0 = (int)floorf(fy);
  b.x1 = min(b.x0 + 1, W - 1); b.y1 = min(b.y0 + 1, H - 1);
  b.wx = fx - (float)b.x0; b.wy = fy - (float)b.y0;
  return b;
}

struct DeformGlobal {
  const float* rot_base;      // [T,P,4] per-frame base quaternions (replace `rotation`) or null
  float* g_rot_base;          // backward: d/d rot_base, [T,P,4], or null
  const float* g_featmean;    // backward: d/d (mean feature of frame t), [T, nfeat], or null
  float* featmean;            // kMode 2: [T, nfeat], pre-zeroed; receives sum / P
};

// kMode: 0 = forward, 2 = per-frame mean of the k-planes features only (backward: deform_backward_kernel)
template <int kMode>
__global__ void __launch_bounds__(128)
deform_kernel(DeformGrids G, DeformMlp M, DeformGlobal X, const float* __restrict__ xyz, const float* __restrict__ scaling,
              const float* __restrict__ rotation, const float* __restrict__ times, int P, int T, int deform_scale,
              float* __restrict__ out_means, float* __restrict__ out_scales, float* __restrict__ out_rots,
              const float* __restrict__ g_means, const float* __restrict__ g_scales, const float* __restrict__ g_rots) {
  constexpr bool kBackward = false;
  static_assert(kMode == 0 || kMode == 2, "backward is a separate kernel");
  extern __shared__ __align__(16) float sm[];
  // shared copies of the MLP weights
  float* sw1 = sm;                                   // [3][32][32]
  float* sw2 = sw1 + 3 * kHid * kHid;                // [3][4][32] (padded to 4 outputs)
  const int nfeat = G.scales * kFeat;
  if (kMode != 2) {
    for (int i = threadIdx.x; i < 3 * kHid * kHid; i += blockDim.x) {
      const int m = i / (kHid * kHid), r = i % (kHid * kHid);
      sw1[i] = (r % kHid < nfeat) ? M.w1[m][(r / kHid) * nfeat + r % kHid] : 0.f;
    }
    for (int i = threadIdx.x; i < 3 * 4 * kHid; i += blockDim.x) {
      const int m = i / (4 * kHid), r = (i % (4 * kHid)) / kHid, c = i % kHid;
      sw2[i] = r < out_dim(m) ? M.w2[m][r * kHid + c] : 0.f;
    }
  } else {
    for (int i = threadIdx.x; i < 2 * kHid; i += blockDim.x) sm[i] = 0.f;   // [2 frames a block may straddle][32]
  }
  __syncthreads();
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  const bool active = idx < P * T;
  const int t = active ? idx / P : 0, i = active ? idx % P : 0;
  float pt[4] = {0.f, 0.f, 0.f, 0.f};
  if (active) { pt[0] = xyz[3 * i]; pt[1] = xyz[3 * i + 1]; pt[2] = xyz[3 * i + 2]; pt[3] = times[t]; }
  // ---- features: product over planes of bilinear samples
  float feat[kHid];
#pragma unroll
  for (int c = 0; c < kHid; ++c) feat[c] = c < nfeat ? 1.f : 0.f;
  if (active) {
    for (int s = 0; s < G.scales; ++s)
      for (int pl = 0; pl < kPlanes; ++pl) {
        const int W = G.w[s][pl], H = G.h[s][pl];
        const Bilerp b = bilerp_setup(pt[c_comb[pl][0]], pt[c_comb[pl][1]], W, H);
        const float* g = G.plane[s][pl];
#pragma unroll
        for (int c = 0; c < kFeat; ++c) {
          const float* gc = g + (size_t)c * H * W;
          const float v00 = __ldg(gc + b.y0 * W + b.x0), v01 = __ldg(gc + b.y0 * W + b.x1);
          const float v10 = __ldg(gc + b.y1 * W + b.x0), v11 = __ldg(gc + b.y1 * W + b.x1);
          const float v = (v00 * (1.f - b.wx) + v01 * b.wx) * (1.f - b.wy) + (v10 * (1.f - b.wx) + v11 * b.wx) * b.wy;
          feat[s * kFeat + c] *= v;
        }
      }
  }
  if (kMode == 2) {
    // block-level sum per frame (a 128-thread block touches at most two frames when P >= 128), then one atomic per value
    const int t_first = (blockIdx.x * blockDim.x) / P;
    if (active) {
      const int slot = t - t_first;
      if (slot < 2) {
#pragma unroll
        for (int c = 0; c < kHid; ++c) if (c < nfeat) atomicAdd(&sm[slot * kHid + c], feat[c]);
      } else {
#pragma unroll
        for (int c = 0; c < kHid; ++c) if (c < nfeat) atomicAdd(&X.featmean[(size_t)t * nfeat + c], feat[c] / (float)P);
      }
    }
    __syncthreads();
    for (int k = threadIdx.x; k < 2 * kHid; k += blockDim.x) {
      const int slot = k / kHid, c = k % kHid;
      if (c < nfeat && t_first + slot < T && sm[k] != 0.f) atomicAdd(&X.featmean[(size_t)(t_first + slot) * nfeat + c], sm[k] / (float)P);
    }
    return;
  }
  // ---- three MLPs
  // the weights are broadcast reads from shared memory: 16-byte loads (4 FMAs per load) -- with scalar loads the kernel sat on
  // the shared-memory pipe (one LDS per FMA: 0.68 ms for 16 frames x 50k gaussians, profiles/r02_splat_launches.txt)
  float outv[3][4];
#pragma unroll 1
  for (int m = 0; m < 3; ++m) {
    float hid[kHid];
#pragma unroll
    for (int r = 0; r < kHid; ++r) {
      float a = 0.f;
      const float4* wr = reinterpret_cast<const float4*>(sw1 + (m * kHid + r) * kHid);
#pragma unroll
      for (int c = 0; c < kHid / 4; ++c) {
        const float4 w4 = wr[c];
        a = fmaf(w4.x, feat[4 * c], a); a = fmaf(w4.y, feat[4 * c + 1], a);
        a = fmaf(w4.z, feat[4 * c + 2], a); a = fmaf(w4.w, feat[4 * c + 3], a);
      }
      hid[r] = fmaxf(a, 0.f);
    }
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      float a = 0.f;
      const float4* wr = reinterpret_cast<const float4*>(sw2 + (m * 4 + r) * kHid);
#pragma unroll
      for (int c = 0; c < kHid / 4; ++c) {
        const float4 w4 = wr[c];
        a = fmaf(w4.x, hid[4 * c], a); a = fmaf(w4.y, hid[4 * c + 1], a);
        a = fmaf(w4.z, hid[4 * c + 2], a); a = fmaf(w4.w, hid[4 * c + 3], a);
      }
      outv[m][r] = a;
    }
  }
  float q[4] = {0.f, 0.f, 0.f, 1.f}, sc[3] = {0.f, 0.f, 0.f};
  float qn = 1.f;
  if (active) {
    const float* qb = X.rot_base ? X.rot_base + 4 * ((size_t)t * P + i) : rotation + 4 * i;
    for (int k = 0; k < 4; ++k) q[k] = qb[k] + outv[1][k];
    qn = fmaxf(sqrtf(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]), 1e-12f);
    for (int k = 0; k < 3; ++k) sc[k] = expf(scaling[3 * i + k] + (deform_scale ? outv[2][k] : 0.f));
  }
  if (!kBackward) {
    if (active) {
      const size_t o = (size_t)t * P + i;
      for (int k = 0; k < 3; ++k) out_means[3 * o + k] = pt[k] + outv[0][k];
      for (int k = 0; k < 3; ++k) out_scales[3 * o + k] = sc[k];
      for (int k = 0; k < 4; ++k) out_rots[4 * o + k] = q[k] / qn;
    }
    return;
  }
  // kMode 1 (backward) lives in deform_backward_kernel below
}


// ---------------------------------------------------------------------------------------------------------------
// Backward (round 2).  The round-1 backward was deform_kernel<1>: every thread pushed its 3 x (32x32 + 4x32) weight-gradient
// outer products into ONE shared copy with shared-memory atomics -- all 128 threads of a block on the same addresses -- and
// recomputed the 5 other planes for every (plane, channel) before 4 scalar global atomics: 33 ms of the 47 ms forward+backward
// render step at BASELINE config 3 (profiles/r02_splat_launches.txt).  Here:
//   * persistent blocks loop over chunks of 128 (frame, gaussian) items; a thread OWNS weight-gradient entries (8 of W1 and
//     3 of W2 per MLP) and accumulates them in registers over all chunks: per chunk the block stages dh / feat / hid / dout in
//     shared memory and every thread runs its entries' dot products over the 128 rows (no atomics); ONE global atomic per
//     entry per block at the very end
//   * plane samples of a channel are loaded once (6 planes x 4 texels) and the "product of the other planes" comes from
//     prefix / suffix products
//   * plane gradients go to a CHANNEL-LAST scratch [H, W, 16]: the 16 channels of a texel are 64 contiguous bytes, written
//     with four red.global.add.v4.f32 per corner instead of 16 scalar atomics on 16 different cache lines (the host
//     wrapper transposes the scratch into the [1, 16, H, W] parameter gradient)
// ---------------------------------------------------------------------------------------------------------------
constexpr int kBwdThreads = 128;
constexpr int kLdS = 36;   // padded row (floats) of the staged [128][32] tiles: 16-byte aligned rows, conflict-free float4 reads
constexpr int kOwn = 8 + 3;   // weight-gradient entries a thread owns per MLP: 8 of W1, 3 of W2

__device__ __forceinline__ void red_add_v4(float* addr, float a, float b, float c, float d) {
  asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(addr), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}

__device__ __forceinline__ float plane_sample(const float* __restrict__ gc, const Bilerp& b, int W) {
  return (__ldg(gc + b.y0 * W + b.x0) * (1.f - b.wx) + __ldg(gc + b.y0 * W + b.x1) * b.wx) * (1.f - b.wy) +
         (__ldg(gc + b.y1 * W + b.x0) * (1.f - b.wx) + __ldg(gc + b.y1 * W + b.x1) * b.wx) * b.wy;
}

__global__ void __launch_bounds__(kBwdThreads, 2)
deform_backward_kernel(DeformGrids G, DeformMlp M, DeformGlobal X, const float* __restrict__ xyz, const float* __restrict__ scaling,
                       const float* __restrict__ rotation, const float* __restrict__ times, int P, int T, int deform_scale,
                       const float* __restrict__ g_means, const float* __restrict__ g_scales, const float* __restrict__ g_rots) {
  extern __shared__ __align__(16) float sm[];
  float* sw1 = sm;                                   // [3][32][32]
  float* sw2 = sw1 + 3 * kHid * kHid;                // [3][4][32]
  float* s_feat = sw2 + 3 * 4 * kHid;                // [128][kLdS]
  float* s_a = s_feat + kBwdThreads * kLdS;          // [128][kLdS]: dh of the current MLP, then hid of the current MLP
  float* s_df = s_a + kBwdThreads * kLdS;            // [128][kLdS]: d loss / d feat, accumulated over the three MLPs
  float* s_do = s_df + kBwdThreads * kLdS;           // [128][4]: dout of the current MLP
  float* s_acc = s_do + kBwdThreads * 4;             // [3][kOwn][128]: the weight-gradient entries each thread owns
  const int nfeat = G.scales * kFeat;
  for (int i = threadIdx.x; i < 3 * kHid * kHid; i += blockDim.x) {
    const int m = i / (kHid * kHid), r = i % (kHid * kHid);
    sw1[i] = (r % kHid < nfeat) ? M.w1[m][(r / kHid) * nfeat + r % kHid] : 0.f;
  }
  for (int i = threadIdx.x; i < 3 * 4 * kHid; i += blockDim.x) {
    const int m = i / (4 * kHid), r = (i % (4 * kHid)) / kHid, c = i % kHid;
    sw2[i] = r < out_dim(m) ? M.w2[m][r * kHid + c] : 0.f;
  }
  for (int i = threadIdx.x; i < 3 * kOwn * kBwdThreads; i += blockDim.x) s_acc[i] = 0.f;
  // weight-gradient entries this thread owns: W1[m][r1][c1 .. c1+7] and W2[m][e / 32][e % 32] for e = tid, tid+128, tid+256
  const int r1 = threadIdx.x >> 2, c1 = (threadIdx.x & 3) * 8;
  __syncthreads();
  const long long total = (long long)P * T;
  for (long long base = (long long)blockIdx.x * kBwdThreads; base < total; base += (long long)gridDim.x * kBwdThreads) {
    const long long idx = base + threadIdx.x;
    const bool active = idx < total;
    const int t = active ? (int)(idx / P) : 0, i = active ? (int)(idx % P) : 0;
    float pt[4] = {0.f, 0.f, 0.f, 0.f};
    if (active) { pt[0] = xyz[3 * i]; pt[1] = xyz[3 * i + 1]; pt[2] = xyz[3 * i + 2]; pt[3] = times[t]; }
    // ---- features
    float feat[kHid];
#pragma unroll
    for (int c = 0; c < kHid; ++c) feat[c] = c < nfeat ? 1.f : 0.f;
    if (active) {
      for (int s = 0; s < G.scales; ++s)
        for (int pl = 0; pl < kPlanes; ++pl) {
          const int W = G.w[s][pl], H = G.h[s][pl];
          const Bilerp b = bilerp_setup(pt[c_comb[pl][0]], pt[c_comb[pl][1]], W, H);
          const float* g = G.plane[s][pl];
#pragma unroll
          for (int c = 0; c < kFeat; ++c) feat[s * kFeat + c] *= plane_sample(g + (size_t)c * H * W, b, W);
        }
    }
    __syncthreads();                                  // previous chunk's readers of the staged tiles are done
#pragma unroll
    for (int c = 0; c < kHid; c += 4) {
      *reinterpret_cast<float4*>(s_feat + threadIdx.x * kLdS + c) = make_float4(feat[c], feat[c + 1], feat[c + 2], feat[c + 3]);
      *reinterpret_cast<float4*>(s_df + threadIdx.x * kLdS + c) = make_float4(0.f, 0.f, 0.f, 0.f);
    }
#pragma unroll 1
    for (int m = 0; m < 3; ++m) {
      // forward of MLP m (hidden layer kept; the output only enters the rotation / scale Jacobians)
      float hid[kHid];
#pragma unroll
      for (int r = 0; r < kHid; ++r) {
        float a = 0.f;
        const float4* wr = reinterpret_cast<const float4*>(sw1 + (m * kHid + r) * kHid);
#pragma unroll
        for (int c = 0; c < kHid / 4; ++c) {
          const float4 w4 = wr[c];
          a = fmaf(w4.x, feat[4 * c], a); a = fmaf(w4.y, feat[4 * c + 1], a);
          a = fmaf(w4.z, feat[4 * c + 2], a); a = fmaf(w4.w, feat[4 * c + 3], a);
        }
        hid[r] = fmaxf(a, 0.f);
      }
      float outv[4], dout[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        float a = 0.f;
#pragma unroll
        for (int c = 0; c < kHid; ++c) a = fmaf(sw2[(m * 4 + r) * kHid + c], hid[c], a);
        outv[r] = a;
      }
      if (active) {
        const size_t o = (size_t)t * P + i;
        if (m == 0) {
          for (int k = 0; k < 3; ++k) dout[k] = g_means ? g_means[3 * o + k] : 0.f;
        } else if (m == 2) {
          if (deform_scale && g_scales)
            for (int k = 0; k < 3; ++k) dout[k] = g_scales[3 * o + k] * expf(scaling[3 * i + k] + outv[k]);           // d exp
        } else if (g_rots) {   // y = q / |q|: dq = (g - y (y.g)) / |q|
          const float* qb = X.rot_base ? X.rot_base + 4 * o : rotation + 4 * i;
          float q[4], y[4], dot = 0.f;
          for (int k = 0; k < 4; ++k) q[k] = qb[k] + outv[k];
          const float qn = fmaxf(sqrtf(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]), 1e-12f);
          for (int k = 0; k < 4; ++k) { y[k] = q[k] / qn; dot += y[k] * g_rots[4 * o + k]; }
          for (int k = 0; k < 4; ++k) dout[k] = (g_rots[4 * o + k] - y[k] * dot) / qn;
          if (X.g_rot_base) for (int k = 0; k < 4; ++k) X.g_rot_base[4 * o + k] = dout[k];   // q = rot_base + delta
        }
      }
      float dh[kHid];
#pragma unroll
      for (int c = 0; c < kHid; ++c) {
        float a = 0.f;
#pragma unroll
        for (int r = 0; r < 4; ++r) a = fmaf(sw2[(m * 4 + r) * kHid + c], dout[r], a);
        dh[c] = hid[c] > 0.f ? a : 0.f;
      }
      __syncthreads();                                // s_a / s_do of the previous MLP consumed
#pragma unroll
      for (int c = 0; c < kHid; c += 4) {
        float4 d4 = *reinterpret_cast<float4*>(s_df + threadIdx.x * kLdS + c);
        float add[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int r = 0; r < kHid; ++r) {
          const float4 w4 = *reinterpret_cast<const float4*>(sw1 + (m * kHid + r) * kHid + c);
          add[0] = fmaf(w4.x, dh[r], add[0]); add[1] = fmaf(w4.y, dh[r], add[1]);
          add[2] = fmaf(w4.z, dh[r], add[2]); add[3] = fmaf(w4.w, dh[r], add[3]);
        }
        d4.x += add[0]; d4.y += add[1]; d4.z += add[2]; d4.w += add[3];
        *reinterpret_cast<float4*>(s_df + threadIdx.x * kLdS + c) = d4;
        *reinterpret_cast<float4*>(s_a + threadIdx.x * kLdS + c) = make_float4(dh[c], dh[c + 1], dh[c + 2], dh[c + 3]);
      }
      __syncthreads();
      {   // W1[m] += dh^T feat over the 128 rows of the chunk: this thread's 8 entries
        float acc[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] = s_acc[(m * kOwn + j) * kBwdThreads + threadIdx.x];
        for (int row = 0; row < kBwdThreads; ++row) {
          const float a = s_a[row * kLdS + r1];
          const float4 f0 = *reinterpret_cast<const float4*>(s_feat + row * kLdS + c1);
          const float4 f1 = *reinterpret_cast<const float4*>(s_feat + row * kLdS + c1 + 4);
          acc[0] = fmaf(a, f0.x, acc[0]); acc[1] = fmaf(a, f0.y, acc[1]); acc[2] = fmaf(a, f0.z, acc[2]); acc[3] = fmaf(a, f0.w, acc[3]);
          acc[4] = fmaf(a, f1.x, acc[4]); acc[5] = fmaf(a, f1.y, acc[5]); acc[6] = fmaf(a, f1.z, acc[6]); acc[7] = fmaf(a, f1.w, acc[7]);
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) s_acc[(m * kOwn + j) * kBwdThreads + threadIdx.x] = acc[j];
      }
      __syncthreads();
#pragma unroll
      for (int c = 0; c < kHid; c += 4)
        *reinterpret_cast<float4*>(s_a + threadIdx.x * kLdS + c) = make_float4(hid[c], hid[c + 1], hid[c + 2], hid[c + 3]);
      *reinterpret_cast<float4*>(s_do + threadIdx.x * 4) = make_float4(dout[0], dout[1], dout[2], dout[3]);
      __syncthreads();
#pragma unroll
      for (int j = 0; j < 3; ++j) {   // W2[m] += dout^T hid: this thread's 3 entries of the [4][32] matrix
        const int e = threadIdx.x + j * kBwdThreads;
        const int r2 = e >> 5, c2 = e & 31;
        float a2 = s_acc[(m * kOwn + 8 + j) * kBwdThreads + threadIdx.x];
        for (int row = 0; row < kBwdThreads; ++row) a2 = fmaf(s_do[row * 4 + r2], s_a[row * kLdS + c2], a2);
        s_acc[(m * kOwn + 8 + j) * kBwdThreads + threadIdx.x] = a2;
      }
    }
    // ---- plane gradients: d sample_p = dfeat * prod_{q != p} sample_q (prefix / suffix products, no division),
    //      four channels at a time -> one 16-byte vector reduction per bilinear corner
    if (active) {
      for (int s = 0; s < G.scales; ++s) {
        if (!G.gplane[s][0]) continue;
        Bilerp bl[kPlanes];
#pragma unroll
        for (int pl = 0; pl < kPlanes; ++pl) bl[pl] = bilerp_setup(pt[c_comb[pl][0]], pt[c_comb[pl][1]], G.w[s][pl], G.h[s][pl]);
#pragma unroll 1
        for (int c0 = 0; c0 < kFeat; c0 += 4) {
          float4 d4 = *reinterpret_cast<const float4*>(s_df + threadIdx.x * kLdS + s * kFeat + c0);
          if (X.g_featmean) {
            const float* gm = X.g_featmean + (size_t)t * nfeat + s * kFeat + c0;
            const float ip = 1.f / (float)P;
            d4.x += gm[0] * ip; d4.y += gm[1] * ip; d4.z += gm[2] * ip; d4.w += gm[3] * ip;
          }
          const float dv[4] = {d4.x, d4.y, d4.z, d4.w};
          float ds[kPlanes][4];
#pragma unroll
          for (int cc = 0; cc < 4; ++cc) {
            float smp[kPlanes];
#pragma unroll
            for (int pl = 0; pl < kPlanes; ++pl)
              smp[pl] = plane_sample(G.plane[s][pl] + (size_t)(c0 + cc) * G.h[s][pl] * G.w[s][pl], bl[pl], G.w[s][pl]);
            float pre = 1.f, suf[kPlanes];
            suf[kPlanes - 1] = 1.f;
#pragma unroll
            for (int pl = kPlanes - 2; pl >= 0; --pl) suf[pl] = suf[pl + 1] * smp[pl + 1];
#pragma unroll
            for (int pl = 0; pl < kPlanes; ++pl) {
              ds[pl][cc] = dv[cc] * pre * suf[pl];
              pre *= smp[pl];
            }
          }
#pragma unroll
          for (int pl = 0; pl < kPlanes; ++pl) {
            const float d0 = ds[pl][0], d1 = ds[pl][1], d2 = ds[pl][2], d3 = ds[pl][3];
            if (d0 == 0.f && d1 == 0.f && d2 == 0.f && d3 == 0.f) continue;
            float* gg = G.gplane[s][pl] + c0;            // channel-last scratch [H][W][16]
            const int W = G.w[s][pl];
            const Bilerp b = bl[pl];
            const float w00 = (1.f - b.wx) * (1.f - b.wy), w01 = b.wx * (1.f - b.wy), w10 = (1.f - b.wx) * b.wy, w11 = b.wx * b.wy;
            red_add_v4(gg + ((size_t)b.y0 * W + b.x0) * kFeat, d0 * w00, d1 * w00, d2 * w00, d3 * w00);
            red_add_v4(gg + ((size_t)b.y0 * W + b.x1) * kFeat, d0 * w01, d1 * w01, d2 * w01, d3 * w01);
            red_add_v4(gg + ((size_t)b.y1 * W + b.x0) * kFeat, d0 * w10, d1 * w10, d2 * w10, d3 * w10);
            red_add_v4(gg + ((size_t)b.y1 * W + b.x1) * kFeat, d0 * w11, d1 * w11, d2 * w11, d3 * w11);
          }
        }
      }
    }
  }
  __syncthreads();
  // ---- one global atomic per owned weight-gradient entry
  for (int m = 0; m < 3; ++m) {
    if (M.gw1[m]) {
      for (int j = 0; j < 8; ++j) {
        const float v = s_acc[(m * kOwn + j) * kBwdThreads + threadIdx.x];
        if (c1 + j < nfeat && v != 0.f) atomicAdd(&M.gw1[m][r1 * nfeat + c1 + j], v);
      }
    }
    if (M.gw2[m]) {
      for (int j = 0; j < 3; ++j) {
        const int e = threadIdx.x + j * kBwdThreads;
        const float v = s_acc[(m * kOwn + 8 + j) * kBwdThreads + threadIdx.x];
        if ((e >> 5) < out_dim(m) && v != 0.f) atomicAdd(&M.gw2[m][(e >> 5) * kHid + (e & 31)], v);
      }
    }
  }
}

}  // namespace a3d

using namespace a3d;

static DeformGlobal globals(const a3d_deform_args* a, float* featmean) {
  DeformGlobal X;
  X.rot_base = a->rot_base; X.g_rot_base = a->grad_rot_base; X.g_featmean = a->grad_featmean; X.featmean = featmean;
  return X;
}

static int fill(const a3d_deform_args* a, DeformGrids* G, DeformMlp* M) {
  const bool bwd = a && a->grad_w1[0] != nullptr;
  (void)bwd;
  if (!a || a->P <= 0 || a->T <= 0) return fail(A3D_EINVAL, "a3d_deform: bad sizes");
  if (a->num_scales < 1 || a->num_scales > kMaxScales || a->channels != kFeat || a->hidden != kHid)
    return fail(A3D_EINVAL, "a3d_deform: supports 1-2 scales x 16 channels and 32-wide MLPs (got %d x %d, hidden %d)", a->num_scales,
                a->channels, a->hidden);
  memset(G, 0, sizeof(*G));
  memset(M, 0, sizeof(*M));
  G->scales = a->num_scales;
  for (int s = 0; s < a->num_scales; ++s)
    for (int p = 0; p < kPlanes; ++p) {
      G->plane[s][p] = a->planes[s * kPlanes + p];
      G->gplane[s][p] = a->grad_planes[s * kPlanes + p];
      G->h[s][p] = a->plane_h[s * kPlanes + p];
      G->w[s][p] = a->plane_w[s * kPlanes + p];
      if (!G->plane[s][p] || G->h[s][p] < 1 || G->w[s][p] < 1) return fail(A3D_EINVAL, "a3d_deform: bad plane %d/%d", s, p);
    }
  for (int m = 0; m < 3; ++m) {
    M->w1[m] = a->w1[m]; M->w2[m] = a->w2[m];
    M->gw1[m] = a->grad_w1[m];
    M->gw2[m] = a->grad_w2[m];
    if (!M->w1[m] || !M->w2[m]) return fail(A3D_EINVAL, "a3d_deform: null MLP weights");
  }
  return 0;
}

extern "C" int a3d_deform_forward(const a3d_deform_args* a, float* means, float* scales, float* rots, void* stream) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  DeformGrids G; DeformMlp M;
  if (int r = fill(a, &G, &M)) return r;
  const int n = a->P * a->T;
  const size_t smem = (3 * kHid * kHid + 3 * 4 * kHid) * sizeof(float);
  deform_kernel<0><<<(n + 127) / 128, 128, smem, st>>>(G, M, globals(a, nullptr), a->xyz, a->scaling, a->rotation, a->times, a->P, a->T,
                                                      a->deform_scale, means, scales, rots, nullptr, nullptr, nullptr);
  A3D_LAUNCH_CHECK();
  return A3D_OK;
}

extern "C" int a3d_deform_featmean(const a3d_deform_args* a, float* featmean, void* stream) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  DeformGrids G; DeformMlp M;
  if (int r = fill(a, &G, &M)) return r;
  if (!featmean) return fail(A3D_EINVAL, "a3d_deform_featmean: null output");
  if (a->P < 128) return fail(A3D_EINVAL, "a3d_deform_featmean: needs at least 128 gaussians (got %d)", a->P);
  const int n = a->P * a->T;
  A3D_CUDA_CHECK(cudaMemsetAsync(featmean, 0, sizeof(float) * a->T * a->num_scales * kFeat, st));
  const size_t smem = (3 * kHid * kHid + 3 * 4 * kHid) * sizeof(float);
  deform_kernel<2><<<(n + 127) / 128, 128, smem, st>>>(G, M, globals(a, featmean), a->xyz, a->scaling, a->rotation, a->times, a->P, a->T,
                                                      a->deform_scale, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr);
  A3D_LAUNCH_CHECK();
  return A3D_OK;
}

extern "C" int a3d_deform_backward(const a3d_deform_args* a, const float* g_means, const float* g_scales, const float* g_rots,
                                   void* stream) {
  // grad_planes[i]: CHANNEL-LAST scratch [H_i, W_i, 16] (zero-initialised by the caller, accumulated into); the caller transposes
  // it into the [1, 16, H, W] parameter gradient (animate3d_b200/gaussian4d.py)
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  DeformGrids G; DeformMlp M;
  if (int r = fill(a, &G, &M)) return r;
  for (int sc = 0; sc < a->num_scales; ++sc) {
    bool any = false, all = true;
    for (int p = 0; p < kPlanes; ++p) { any = any || G.gplane[sc][p]; all = all && G.gplane[sc][p]; }
    if (any != all) return fail(A3D_EINVAL, "a3d_deform_backward: plane gradients of a scale must be all set or all null");
    for (int p = 0; p < kPlanes; ++p)
      if (G.gplane[sc][p] && (reinterpret_cast<uintptr_t>(G.gplane[sc][p]) & 15))
        return fail(A3D_EINVAL, "a3d_deform_backward: plane gradient scratch must be 16-byte aligned");
  }
  const long long n = (long long)a->P * a->T;
  const size_t smem = (3 * kHid * kHid + 3 * 4 * kHid + 3 * kBwdThreads * kLdS + kBwdThreads * 4 + 3 * kOwn * kBwdThreads) * sizeof(float);
  static bool attr = false;
  static int sms = 0;
  if (!attr) {
    A3D_CUDA_CHECK(cudaFuncSetAttribute(deform_backward_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    attr = true;
  }
  long long blocks = (n + kBwdThreads - 1) / kBwdThreads;
  if (blocks > 2ll * sms) blocks = 2ll * sms;          // persistent: 2 blocks (86 KB shared each) per SM
  deform_backward_kernel<<<(unsigned)blocks, kBwdThreads, smem, st>>>(G, M, globals(a, nullptr), a->xyz, a->scaling, a->rotation, a->times,
                                                                     a->P, a->T, a->deform_scale, g_means, g_scales, g_rots);
  A3D_LAUNCH_CHECK();
  return A3D_OK;
}
