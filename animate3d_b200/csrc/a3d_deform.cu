// Per-frame deformation field of the 4D gaussians, all frames of a batch in one launch:
//   k-planes (HexPlane) lookup -- 2 scales x 6 planes, bilinear, border clamp, align_corners -- product over planes, concat
//   over scales -> 32 features -> three bias-free MLPs 32 -> 32 (ReLU) -> {3, 4, 3} -> xyz + d, exp(s + d), normalize(q + d)
// forward and backward (gradients to the plane grids and MLP weights; the static gaussians are frozen buffers in
// Animate3D, gaussian_4d.py:262-297).  The `use_global_trans` branch (gaussian_4d.py:499-511, 525-539) needs the MEAN feature
// vector of a frame before any output can be formed: deform_featmean_kernel computes those means (one extra pass over the
// L2-resident planes, summed in a fixed order), the host evaluates the two 32-wide global MLPs + Euler matrix on [T, 32],
// and the main pass takes the rotated base quaternions as `rot_base`; backward returns d/d rot_base and folds d/d mean-feature back into the plane gradients.  Replaces, per (frame, gaussian), the 12 grid_sample + 6 GEMM + elementwise launches the
// reference issues PER CAMERA (custom/threestudio-animate3d/geometry/gaussian_4d.py:39-64, 450-548;
// renderer/diff_gaussian_rasterizer_advanced_4d.py:77-83, 119-135) and de-duplicates the 4 views of a frame.
#include <cooperative_groups.h>

#include "a3d_host.cuh"
#include "a3d_segsort.cuh"

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

// coordinates (x, y, z, t) of each plane, the first one indexing W.  One list: kernels read c_comb, the host (which cannot
// read __constant__ memory) kComb when it launches the per-plane gather of the fixed-order backward.
#define A3D_PLANE_AXES {{0, 1}, {0, 2}, {0, 3}, {1, 2}, {1, 3}, {2, 3}}
__device__ __constant__ int c_comb[kPlanes][2] = A3D_PLANE_AXES;
constexpr int kComb[kPlanes][2] = A3D_PLANE_AXES;
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
};

__device__ __forceinline__ float plane_sample(const float* __restrict__ gc, const Bilerp& b, int W) {
  return (__ldg(gc + b.y0 * W + b.x0) * (1.f - b.wx) + __ldg(gc + b.y0 * W + b.x1) * b.wx) * (1.f - b.wy) +
         (__ldg(gc + b.y1 * W + b.x0) * (1.f - b.wx) + __ldg(gc + b.y1 * W + b.x1) * b.wx) * b.wy;
}

// (x, y, z, t) of item idx = frame t * P + gaussian i; an inactive item is (0, 0, 0, 0) with t = i = 0
template <class Idx>
__device__ __forceinline__ void item_point(const float* __restrict__ xyz, const float* __restrict__ times, int P, Idx idx, bool active,
                                           float (&pt)[4], int& t, int& i) {
  t = active ? (int)(idx / (Idx)P) : 0;
  i = active ? (int)(idx % (Idx)P) : 0;
  pt[0] = pt[1] = pt[2] = pt[3] = 0.f;
  if (active) { pt[0] = xyz[3 * i]; pt[1] = xyz[3 * i + 1]; pt[2] = xyz[3 * i + 2]; pt[3] = times[t]; }
}

// k-planes feature of point pt: per scale, the product over the 6 planes of the bilinear samples of the 16 channels.
// Channels >= nfeat are 0; an inactive item reads nothing and keeps 1 in the others.
__device__ __forceinline__ void kplanes_feature(const DeformGrids& G, const float (&pt)[4], bool active, float (&feat)[kHid]) {
  const int nfeat = G.scales * kFeat;
#pragma unroll
  for (int c = 0; c < kHid; ++c) feat[c] = c < nfeat ? 1.f : 0.f;
  if (!active) return;
  for (int s = 0; s < G.scales; ++s)
    for (int pl = 0; pl < kPlanes; ++pl) {
      const int W = G.w[s][pl], H = G.h[s][pl];
      const Bilerp b = bilerp_setup(pt[c_comb[pl][0]], pt[c_comb[pl][1]], W, H);
#pragma unroll
      for (int c = 0; c < kFeat; ++c) feat[s * kFeat + c] *= plane_sample(G.plane[s][pl] + (size_t)c * H * W, b, W);
    }
}

// MLP weights into shared memory: sw1 [3][32][32] (input columns >= nfeat zeroed), sw2 [3][4][32] (padded to 4 outputs)
__device__ __forceinline__ void stage_mlp_weights(const DeformMlp& M, int nfeat, float* sw1, float* sw2) {
  for (int i = threadIdx.x; i < 3 * kHid * kHid; i += blockDim.x) {
    const int m = i / (kHid * kHid), r = i % (kHid * kHid);
    sw1[i] = (r % kHid < nfeat) ? M.w1[m][(r / kHid) * nfeat + r % kHid] : 0.f;
  }
  for (int i = threadIdx.x; i < 3 * 4 * kHid; i += blockDim.x) {
    const int m = i / (4 * kHid), r = (i % (4 * kHid)) / kHid, c = i % kHid;
    sw2[i] = r < out_dim(m) ? M.w2[m][r * kHid + c] : 0.f;
  }
}

// MLP m on the staged weights: hid = relu(W1 feat), out = W2 hid.  The weights are broadcast reads from shared memory:
// 16-byte loads (4 FMAs per load) -- with scalar loads the forward sat on the shared-memory pipe (one LDS per FMA: 0.68 ms
// for 16 frames x 50k gaussians, profiles/r02_splat_launches.txt)
__device__ __forceinline__ void mlp_forward(const float* sw1, const float* sw2, int m, const float (&feat)[kHid], float (&hid)[kHid],
                                            float (&out)[4]) {
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
    out[r] = a;
  }
}

// y = (qb + d) / max(|qb + d|, 1e-12); returns the clamped norm
__device__ __forceinline__ float normalized_rotation(const float* qb, const float* d, float (&y)[4]) {
  float q[4];
  for (int k = 0; k < 4; ++k) q[k] = qb[k] + d[k];
  const float qn = fmaxf(sqrtf(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]), 1e-12f);
  for (int k = 0; k < 4; ++k) y[k] = q[k] / qn;
  return qn;
}

__global__ void __launch_bounds__(128)
deform_kernel(DeformGrids G, DeformMlp M, DeformGlobal X, const float* __restrict__ xyz, const float* __restrict__ scaling,
              const float* __restrict__ rotation, const float* __restrict__ times, int P, int T, int deform_scale,
              float* __restrict__ out_means, float* __restrict__ out_scales, float* __restrict__ out_rots) {
  extern __shared__ __align__(16) float sm[];
  float* sw1 = sm;
  float* sw2 = sw1 + 3 * kHid * kHid;
  stage_mlp_weights(M, G.scales * kFeat, sw1, sw2);
  __syncthreads();
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  const bool active = idx < P * T;
  int t, i;
  float pt[4];
  item_point(xyz, times, P, idx, active, pt, t, i);
  float feat[kHid];
  kplanes_feature(G, pt, active, feat);
  float outv[3][4];
#pragma unroll 1
  for (int m = 0; m < 3; ++m) {
    float hid[kHid];
    mlp_forward(sw1, sw2, m, feat, hid, outv[m]);
  }
  if (active) {
    const size_t o = (size_t)t * P + i;
    float y[4];
    normalized_rotation(X.rot_base ? X.rot_base + 4 * o : rotation + 4 * i, outv[1], y);
    for (int k = 0; k < 3; ++k) out_means[3 * o + k] = pt[k] + outv[0][k];
    for (int k = 0; k < 3; ++k) out_scales[3 * o + k] = expf(scaling[3 * i + k] + (deform_scale ? outv[2][k] : 0.f));
    for (int k = 0; k < 4; ++k) out_rots[4 * o + k] = y[k];
  }
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

// Per-frame mean feature in a fixed order: a cluster of kFmCtas CTAs per frame; each thread sums a strided subset of the
// gaussians, each CTA sums its threads in thread order, and CTA rank 0 adds the cluster's CTA sums in rank order through
// distributed shared memory.  No atomics and no scratch: bit-reproducible for a given launch geometry.
constexpr int kFmCtas = 8, kFmThreads = 256;

__global__ void __cluster_dims__(kFmCtas, 1, 1) __launch_bounds__(kFmThreads)
deform_featmean_kernel(DeformGrids G, const float* __restrict__ xyz, const float* __restrict__ times, int P, float* __restrict__ featmean) {
  namespace cg = cooperative_groups;
  cg::cluster_group cluster = cg::this_cluster();
  __shared__ float s_rows[kFmThreads][kHid + 1];
  __shared__ float s_cta[kHid];
  const int rank = (int)cluster.block_rank(), t = blockIdx.y, nfeat = G.scales * kFeat;
  float acc[kHid];
#pragma unroll
  for (int c = 0; c < kHid; ++c) acc[c] = 0.f;
  const float tm = times[t];
  for (int i = rank * kFmThreads + threadIdx.x; i < P; i += kFmCtas * kFmThreads) {
    const float pt[4] = {xyz[3 * i], xyz[3 * i + 1], xyz[3 * i + 2], tm};
    float feat[kHid];
    kplanes_feature(G, pt, true, feat);
#pragma unroll
    for (int c = 0; c < kHid; ++c) acc[c] += feat[c];
  }
#pragma unroll
  for (int c = 0; c < kHid; ++c) s_rows[threadIdx.x][c] = acc[c];
  __syncthreads();
  if (threadIdx.x < kHid) {
    float a = 0.f;
    for (int r = 0; r < kFmThreads; ++r) a += s_rows[r][threadIdx.x];
    s_cta[threadIdx.x] = a;
  }
  cluster.sync();
  if (rank == 0 && threadIdx.x < nfeat) {
    float a = 0.f;
    for (int r = 0; r < kFmCtas; ++r) a += cluster.map_shared_rank(s_cta, r)[threadIdx.x];
    featmean[(size_t)t * nfeat + threadIdx.x] = a / (float)P;
  }
  cluster.sync();   // the other CTAs' shared memory must outlive rank 0's reads
}

// kDet: plane gradients are not scattered; every (scale, plane, frame, gaussian) stores its 16-channel factor
// (d loss / d feature x product of the other planes' samples) to fac[plane][point][16], and the per-thread weight-gradient
// entries go to part[CTA][...] instead of global atomics
template <bool kDet>
__global__ void __launch_bounds__(kBwdThreads, 2)
deform_backward_kernel(DeformGrids G, DeformMlp M, DeformGlobal X, const float* __restrict__ xyz, const float* __restrict__ scaling,
                       const float* __restrict__ rotation, const float* __restrict__ times, int P, int T, int deform_scale,
                       const float* __restrict__ g_means, const float* __restrict__ g_scales, const float* __restrict__ g_rots,
                       float* __restrict__ fac, float* __restrict__ part) {
  extern __shared__ __align__(16) float sm[];
  float* sw1 = sm;                                   // [3][32][32]
  float* sw2 = sw1 + 3 * kHid * kHid;                // [3][4][32]
  float* s_feat = sw2 + 3 * 4 * kHid;                // [128][kLdS]
  float* s_a = s_feat + kBwdThreads * kLdS;          // [128][kLdS]: dh of the current MLP, then hid of the current MLP
  float* s_df = s_a + kBwdThreads * kLdS;            // [128][kLdS]: d loss / d feat, accumulated over the three MLPs
  float* s_do = s_df + kBwdThreads * kLdS;           // [128][4]: dout of the current MLP
  float* s_acc = s_do + kBwdThreads * 4;             // [3][kOwn][128]: the weight-gradient entries each thread owns
  const int nfeat = G.scales * kFeat;
  stage_mlp_weights(M, nfeat, sw1, sw2);
  for (int i = threadIdx.x; i < 3 * kOwn * kBwdThreads; i += blockDim.x) s_acc[i] = 0.f;
  // weight-gradient entries this thread owns: W1[m][r1][c1 .. c1+7] and W2[m][e / 32][e % 32] for e = tid, tid+128, tid+256
  const int r1 = threadIdx.x >> 2, c1 = (threadIdx.x & 3) * 8;
  __syncthreads();
  const long long total = (long long)P * T;
  for (long long base = (long long)blockIdx.x * kBwdThreads; base < total; base += (long long)gridDim.x * kBwdThreads) {
    const long long idx = base + threadIdx.x;
    const bool active = idx < total;
    int t, i;
    float pt[4];
    item_point(xyz, times, P, idx, active, pt, t, i);
    float feat[kHid];
    kplanes_feature(G, pt, active, feat);
    __syncthreads();                                  // previous chunk's readers of the staged tiles are done
#pragma unroll
    for (int c = 0; c < kHid; c += 4) {
      *reinterpret_cast<float4*>(s_feat + threadIdx.x * kLdS + c) = make_float4(feat[c], feat[c + 1], feat[c + 2], feat[c + 3]);
      *reinterpret_cast<float4*>(s_df + threadIdx.x * kLdS + c) = make_float4(0.f, 0.f, 0.f, 0.f);
    }
#pragma unroll 1
    for (int m = 0; m < 3; ++m) {
      // forward of MLP m (hidden layer kept; the output only enters the rotation / scale Jacobians)
      float hid[kHid], outv[4], dout[4] = {0.f, 0.f, 0.f, 0.f};
      mlp_forward(sw1, sw2, m, feat, hid, outv);
      if (active) {
        const size_t o = (size_t)t * P + i;
        if (m == 0) {
          for (int k = 0; k < 3; ++k) dout[k] = g_means ? g_means[3 * o + k] : 0.f;
        } else if (m == 2) {
          if (deform_scale && g_scales)
            for (int k = 0; k < 3; ++k) dout[k] = g_scales[3 * o + k] * expf(scaling[3 * i + k] + outv[k]);           // d exp
        } else if (g_rots) {   // y = q / |q|: dq = (g - y (y.g)) / |q|
          float y[4], dot = 0.f;
          const float qn = normalized_rotation(X.rot_base ? X.rot_base + 4 * o : rotation + 4 * i, outv, y);
          for (int k = 0; k < 4; ++k) dot += y[k] * g_rots[4 * o + k];
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
          if (kDet) {
#pragma unroll
            for (int pl = 0; pl < kPlanes; ++pl)
              *reinterpret_cast<float4*>(fac + ((size_t)(s * kPlanes + pl) * total + idx) * kFeat + c0) =
                  make_float4(ds[pl][0], ds[pl][1], ds[pl][2], ds[pl][3]);
            continue;
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
  if (kDet) {   // this CTA's partials, reduced in CTA order by deform_wgrad_reduce_kernel
    for (int e = threadIdx.x; e < 3 * kOwn * kBwdThreads; e += kBwdThreads) part[(size_t)blockIdx.x * 3 * kOwn * kBwdThreads + e] = s_acc[e];
    return;
  }
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

// entry e of the [3][kOwn][kBwdThreads] partials: MLP m, owned slot j of thread tid (see deform_backward_kernel)
__global__ void deform_wgrad_reduce_kernel(DeformMlp M, const float* __restrict__ part, int ctas, int nfeat) {
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= 3 * kOwn * kBwdThreads) return;
  float a = 0.f;
  for (int b = 0; b < ctas; ++b) a += part[(size_t)b * 3 * kOwn * kBwdThreads + e];
  const int m = e / (kOwn * kBwdThreads), j = (e / kBwdThreads) % kOwn, tid = e % kBwdThreads;
  if (j < 8) {
    const int r1 = tid >> 2, c1 = (tid & 3) * 8;
    if (M.gw1[m] && c1 + j < nfeat) M.gw1[m][r1 * nfeat + c1 + j] += a;
  } else {
    const int ee = tid + (j - 8) * kBwdThreads;
    if (M.gw2[m] && (ee >> 5) < out_dim(m)) M.gw2[m][(ee >> 5) * kHid + (ee & 31)] += a;
  }
}

// key of point idx for one plane: its lower-left cell y0 * W + x0
__global__ void deform_cell_keys_kernel(const float* __restrict__ xyz, const float* __restrict__ times, int P, long long total, int ca,
                                        int cb, int W, int H, uint32_t* __restrict__ keys, uint32_t* __restrict__ vals) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  int t, i;
  float pt[4];
  item_point(xyz, times, P, idx, true, pt, t, i);
  const Bilerp b = bilerp_setup(pt[ca], pt[cb], W, H);
  keys[idx] = (uint32_t)(b.y0 * W + b.x0);
  vals[idx] = (uint32_t)idx;
}

// gradient of texel (y, x), 4 channels per thread: the points of cells (y-1, x-1), (y-1, x), (y, x-1), (y, x) in that order,
// each cell's points in their stable sorted order; a point's weight on this texel is its bilinear weight of the matching corner
__global__ void deform_plane_gather_kernel(const float* __restrict__ xyz, const float* __restrict__ times, int P, int ca, int cb,
                                           int W, int H, const uint2* __restrict__ ranges, const uint32_t* __restrict__ pts,
                                           const float* __restrict__ fac, float* __restrict__ gplane) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= H * W * 4) return;
  const int c0 = (idx & 3) * 4, texel = idx >> 2, y = texel / W, x = texel % W;
  float a[4] = {0.f, 0.f, 0.f, 0.f};
  for (int cy = y - 1; cy <= y; ++cy)
    for (int cx = x - 1; cx <= x; ++cx) {
      if (cy < 0 || cx < 0) continue;
      const uint2 r = ranges[cy * W + cx];
      for (uint32_t k = r.x; k < r.y; ++k) {
        const uint32_t p = pts[k];
        int t, i;
        float pt[4];
        item_point(xyz, times, P, p, true, pt, t, i);
        const Bilerp b = bilerp_setup(pt[ca], pt[cb], W, H);
        // corner (y1, x1) of a cell on the last row / column coincides with (y0, x0) and has weight 0 there
        const float w = (cy == y ? 1.f - b.wy : b.wy) * (cx == x ? 1.f - b.wx : b.wx);
        const float4 f = *reinterpret_cast<const float4*>(fac + (size_t)p * kFeat + c0);
        a[0] += f.x * w; a[1] += f.y * w; a[2] += f.z * w; a[3] += f.w * w;
      }
    }
  float4* dst = reinterpret_cast<float4*>(gplane + (size_t)texel * kFeat + c0);
  float4 v = *dst;
  v.x += a[0]; v.y += a[1]; v.z += a[2]; v.w += a[3];
  *dst = v;
}

}  // namespace a3d

using namespace a3d;

static DeformGlobal globals(const a3d_deform_args* a) {
  DeformGlobal X;
  X.rot_base = a->rot_base; X.g_rot_base = a->grad_rot_base; X.g_featmean = a->grad_featmean;
  return X;
}

static int fill(const a3d_deform_args* a, DeformGrids* G, DeformMlp* M) {
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
  deform_kernel<<<(n + 127) / 128, 128, smem, st>>>(G, M, globals(a), a->xyz, a->scaling, a->rotation, a->times, a->P, a->T,
                                                   a->deform_scale, means, scales, rots);
  A3D_LAUNCH_CHECK();
  return A3D_OK;
}

extern "C" int a3d_deform_featmean(const a3d_deform_args* a, float* featmean, void* stream) {
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  DeformGrids G; DeformMlp M;
  if (int r = fill(a, &G, &M)) return r;
  if (!featmean) return fail(A3D_EINVAL, "a3d_deform_featmean: null output");
  if (a->T > 65535) return fail(A3D_EINVAL, "a3d_deform_featmean: at most 65535 frames (got %d)", a->T);
  deform_featmean_kernel<<<dim3(kFmCtas, a->T), kFmThreads, 0, st>>>(G, a->xyz, a->times, a->P, featmean);
  A3D_LAUNCH_CHECK();
  return A3D_OK;
}

// ---- backward
constexpr size_t kBwdSmem = (3 * kHid * kHid + 3 * 4 * kHid + 3 * kBwdThreads * kLdS + kBwdThreads * 4 + 3 * kOwn * kBwdThreads) * sizeof(float);

static long long backward_ctas(long long n) {
  long long blocks = (n + kBwdThreads - 1) / kBwdThreads;
  const long long cap = 2ll * sm_count();              // persistent: 2 blocks (86 KB shared each) per SM
  return blocks > cap ? cap : blocks;
}

struct DeformDetScratch {
  float* fac;                    // [num_scales * 6][T * P][16]
  float* part;                   // [ctas][3 * kOwn * kBwdThreads]
  uint32_t *keys_in, *vals_in, *keys_out, *vals_out;   // [T * P]
  uint2* ranges;                 // [largest plane's H * W]
  void* temp;
  size_t temp_bytes;
};

static size_t carve_det(void* base, const a3d_deform_args* a, DeformDetScratch* s) {
  Carve c{static_cast<char*>(base)};
  const size_t n = (size_t)a->P * a->T;
  uint32_t cells = 1;
  for (int p = 0; p < a->num_scales * kPlanes; ++p) {
    const uint32_t hw = (uint32_t)a->plane_h[p] * (uint32_t)a->plane_w[p];
    if (hw > cells) cells = hw;
  }
  DeformDetScratch w;
  w.fac = c.take<float>((size_t)a->num_scales * kPlanes * n * kFeat);
  w.part = c.take<float>((size_t)backward_ctas((long long)n) * 3 * kOwn * kBwdThreads);
  w.keys_in = c.take<uint32_t>(n);
  w.vals_in = c.take<uint32_t>(n);
  w.keys_out = c.take<uint32_t>(n);
  w.vals_out = c.take<uint32_t>(n);
  w.ranges = c.take<uint2>(cells);
  w.temp_bytes = seg_sort_temp_bytes((int)n, cells);
  w.temp = c.take<char>(w.temp_bytes);
  if (s) *s = w;
  return c.bytes();
}

extern "C" size_t a3d_deform_backward_scratch_bytes(const a3d_deform_args* a) {
  DeformGrids G; DeformMlp M;
  if (!a || !a->deterministic || fill(a, &G, &M)) return 0;
  return carve_det(nullptr, a, nullptr);
}

extern "C" int a3d_deform_backward(const a3d_deform_args* a, const float* g_means, const float* g_scales, const float* g_rots,
                                   void* scratch, size_t scratch_bytes, void* stream) {
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
  const bool det = a->deterministic != 0;
  DeformDetScratch s{};
  if (det) {
    if (n > 0x7fffffffll) return fail(A3D_EINVAL, "a3d_deform_backward: T * P too large for the deterministic path");
    const size_t need = carve_det(scratch, a, &s);
    if (!scratch || scratch_bytes < need) return fail(A3D_EINVAL, "a3d_deform_backward: deterministic scratch %zu < %zu bytes", scratch_bytes, need);
  }
  static bool attr = false;
  if (!attr) {
    A3D_CUDA_CHECK(cudaFuncSetAttribute(deform_backward_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kBwdSmem));
    A3D_CUDA_CHECK(cudaFuncSetAttribute(deform_backward_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kBwdSmem));
    attr = true;
  }
  const long long blocks = backward_ctas(n);
  if (!det) {
    deform_backward_kernel<false><<<(unsigned)blocks, kBwdThreads, kBwdSmem, st>>>(G, M, globals(a), a->xyz, a->scaling, a->rotation,
                                                                                  a->times, a->P, a->T, a->deform_scale, g_means, g_scales,
                                                                                  g_rots, nullptr, nullptr);
    A3D_LAUNCH_CHECK();
    return A3D_OK;
  }
  deform_backward_kernel<true><<<(unsigned)blocks, kBwdThreads, kBwdSmem, st>>>(G, M, globals(a), a->xyz, a->scaling, a->rotation,
                                                                               a->times, a->P, a->T, a->deform_scale, g_means, g_scales,
                                                                               g_rots, s.fac, s.part);
  A3D_LAUNCH_CHECK();
  deform_wgrad_reduce_kernel<<<(3 * kOwn * kBwdThreads + 255) / 256, 256, 0, st>>>(M, s.part, (int)blocks, G.scales * kFeat);
  A3D_LAUNCH_CHECK();
  for (int sc = 0; sc < G.scales; ++sc) {
    if (!G.gplane[sc][0]) continue;
    for (int pl = 0; pl < kPlanes; ++pl) {
      const int W = G.w[sc][pl], H = G.h[sc][pl], ca = kComb[pl][0], cb = kComb[pl][1];
      deform_cell_keys_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(a->xyz, a->times, a->P, n, ca, cb, W, H, s.keys_in, s.vals_in);
      A3D_LAUNCH_CHECK();
      if (int r = seg_sort(s.keys_in, s.vals_in, s.keys_out, s.vals_out, (int)n, (uint32_t)(H * W), s.ranges, s.temp, s.temp_bytes, st))
        return r;
      deform_plane_gather_kernel<<<(H * W * 4 + 255) / 256, 256, 0, st>>>(a->xyz, a->times, a->P, ca, cb, W, H, s.ranges, s.vals_out,
                                                                          s.fac + (size_t)(sc * kPlanes + pl) * n * kFeat, G.gplane[sc][pl]);
      A3D_LAUNCH_CHECK();
    }
  }
  return A3D_OK;
}
