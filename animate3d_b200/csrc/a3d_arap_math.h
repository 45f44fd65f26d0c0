// ARAP regulariser arithmetic shared by the CUDA kernel (a3d_arap.cu) and the CPU harness (tests/cpu_harness/arap_cpu.cpp):
// per (frame t >= 1, node i) the weighted Procrustes rotation of the node's frame-0 edges onto its frame-t edges, the edge
// energy and its gradient.  Reference: custom/threestudio-animate3d/systems/util.py:138-173 (estimate_rotation: torch.svd +
// reflection fix) and 183-215 (cal_arap_error; the rotation carries no gradient).
//
// The reference's R = V U'^T (U' = U with the column of the smallest singular value flipped when det <= 0) is THE proper
// rotation maximising sum_n w_n t_n . (R s_n).  It is computed here without an SVD: Horn's closed form -- the eigenvector
// of the largest eigenvalue of the symmetric 4x4 matrix N(S) is the unit quaternion of that rotation -- with a cyclic
// Jacobi eigen-solver (fixed 8 sweeps, no data-dependent branches besides the rotation guard).
#pragma once
#include <math.h>
#include <stdint.h>

#if defined(__CUDACC__)
#define A3D_HD __host__ __device__ __forceinline__
#else
#define A3D_HD inline
#endif

namespace a3d {

constexpr int kArapMaxK = 12;   // the reference's default K is 10 (systems/util.py:58, 183); shipped configs use 3

// eigenvector (w, x, y, z) of the largest eigenvalue of the symmetric 4x4 matrix a (destroyed)
A3D_HD void sym4_max_eigvec(float (&a)[4][4], float (&q)[4]) {
  float v[4][4] = {{1, 0, 0, 0}, {0, 1, 0, 0}, {0, 0, 1, 0}, {0, 0, 0, 1}};
  for (int sweep = 0; sweep < 8; ++sweep) {
    for (int p = 0; p < 3; ++p)
      for (int r = p + 1; r < 4; ++r) {
        const float apq = a[p][r];
        if (fabsf(apq) < 1e-30f) continue;
        const float theta = (a[r][r] - a[p][p]) / (2.0f * apq);
        const float t = (theta >= 0.f ? 1.0f : -1.0f) / (fabsf(theta) + sqrtf(theta * theta + 1.0f));
        const float c = 1.0f / sqrtf(t * t + 1.0f), s = t * c;
        for (int k = 0; k < 4; ++k) {          // A <- A J   (columns p, r)
          const float akp = a[k][p], akr = a[k][r];
          a[k][p] = c * akp - s * akr;
          a[k][r] = s * akp + c * akr;
        }
        for (int k = 0; k < 4; ++k) {          // A <- J^T A (rows p, r)
          const float apk = a[p][k], ark = a[r][k];
          a[p][k] = c * apk - s * ark;
          a[r][k] = s * apk + c * ark;
        }
        for (int k = 0; k < 4; ++k) {
          const float vkp = v[k][p], vkr = v[k][r];
          v[k][p] = c * vkp - s * vkr;
          v[k][r] = s * vkp + c * vkr;
        }
      }
  }
  int best = 0;
  for (int k = 1; k < 4; ++k)
    if (a[k][k] > a[best][best]) best = k;
  for (int k = 0; k < 4; ++k) q[k] = v[k][best];
}

// Rotation R (row-major 3x3) with R s_n ~ t_n from S[a][b] = sum_n w_n s_n[a] t_n[b]; identity when S == 0.
A3D_HD void rotation_from_covariance(const float (&S)[3][3], float (&R)[9]) {
  float norm = 0.f;
  for (int a = 0; a < 3; ++a)
    for (int b = 0; b < 3; ++b) norm += S[a][b] * S[a][b];
  if (!(norm > 0.f)) {
    R[0] = 1; R[1] = 0; R[2] = 0; R[3] = 0; R[4] = 1; R[5] = 0; R[6] = 0; R[7] = 0; R[8] = 1;
    return;
  }
  float N[4][4];
  N[0][0] = S[0][0] + S[1][1] + S[2][2];
  N[0][1] = S[1][2] - S[2][1]; N[0][2] = S[2][0] - S[0][2]; N[0][3] = S[0][1] - S[1][0];
  N[1][1] = S[0][0] - S[1][1] - S[2][2]; N[1][2] = S[0][1] + S[1][0]; N[1][3] = S[2][0] + S[0][2];
  N[2][2] = -S[0][0] + S[1][1] - S[2][2]; N[2][3] = S[1][2] + S[2][1];
  N[3][3] = -S[0][0] - S[1][1] + S[2][2];
  for (int a = 0; a < 4; ++a)
    for (int b = 0; b < a; ++b) N[a][b] = N[b][a];
  float q[4];
  sym4_max_eigvec(N, q);
  const float inv = 1.0f / sqrtf(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
  const float w = q[0] * inv, x = q[1] * inv, y = q[2] * inv, z = q[3] * inv;
  R[0] = 1 - 2 * (y * y + z * z); R[1] = 2 * (x * y - w * z);     R[2] = 2 * (x * z + w * y);
  R[3] = 2 * (x * y + w * z);     R[4] = 1 - 2 * (x * x + z * z); R[5] = 2 * (y * z - w * x);
  R[6] = 2 * (x * z - w * y);     R[7] = 2 * (y * z + w * x);     R[8] = 1 - 2 * (x * x + y * y);
}

// Edges of node i at frame t (nodes [Nt,Nv,3], nbr [Nv,K]): for n < K with j = nbr[i,n] in [0, Nv) (valid[n]),
// e0[n] = x_0[i] - x_0[j] and et[n] = x_t[i] - x_t[j]; w[n] = weight[i,n], or 1 on valid edges when weight is null (the
// reference's call).  Absent edges and n >= K get zero edges; n >= K also zero weight.
A3D_HD void arap_gather(const float* nodes, int Nv, const int* nbr, int K, const float* weight, int i, int t, float (*e0)[3],
                        float (*et)[3], float* w, bool* valid) {
  const float* p0 = nodes;
  const float* pt = nodes + (int64_t)t * Nv * 3;
#pragma unroll
  for (int n = 0; n < kArapMaxK; ++n) {
    const int j = n < K ? nbr[(int64_t)i * K + n] : -1;
    valid[n] = j >= 0 && j < Nv;
    w[n] = (n < K) ? (weight ? weight[(int64_t)i * K + n] : (valid[n] ? 1.f : 0.f)) : 0.f;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      e0[n][c] = valid[n] ? p0[3 * (int64_t)i + c] - p0[3 * (int64_t)j + c] : 0.f;
      et[n][c] = valid[n] ? pt[3 * (int64_t)i + c] - pt[3 * (int64_t)j + c] : 0.f;
    }
  }
}

// One (frame, node): edges e0[n] = p0_i - p0_j(n), et[n] = pt_i - pt_j(n) for the present neighbours (valid[n]), weights w[n].
// Returns the energy sum_n w_n |et_n - R e0_n|^2; g_t[n] / g_0[n] receive d energy / d et_n and d energy / d e0_n (R held
// constant, as in the reference's torch.no_grad around estimate_rotation).
A3D_HD float arap_node(int K, const float (*e0)[3], const float (*et)[3], const bool* valid, const float* w, float (*g_t)[3],
                       float (*g_0)[3]) {
  float S[3][3] = {{0, 0, 0}, {0, 0, 0}, {0, 0, 0}};
  bool same_axis[3] = {true, true, true};      // util.py:152-153: any coordinate whose K edge components are all unchanged
  for (int n = 0; n < K; ++n) {
    const float s0 = valid[n] ? e0[n][0] : 0.f, s1 = valid[n] ? e0[n][1] : 0.f, s2 = valid[n] ? e0[n][2] : 0.f;
    const float t0 = valid[n] ? et[n][0] : 0.f, t1 = valid[n] ? et[n][1] : 0.f, t2 = valid[n] ? et[n][2] : 0.f;
    same_axis[0] = same_axis[0] && (s0 == t0);
    same_axis[1] = same_axis[1] && (s1 == t1);
    same_axis[2] = same_axis[2] && (s2 == t2);
    const float wn = w[n];
    S[0][0] += wn * s0 * t0; S[0][1] += wn * s0 * t1; S[0][2] += wn * s0 * t2;
    S[1][0] += wn * s1 * t0; S[1][1] += wn * s1 * t1; S[1][2] += wn * s1 * t2;
    S[2][0] += wn * s2 * t0; S[2][1] += wn * s2 * t1; S[2][2] += wn * s2 * t2;
  }
  if (same_axis[0] || same_axis[1] || same_axis[2]) {
    for (int a = 0; a < 3; ++a)
      for (int b = 0; b < 3; ++b) S[a][b] = 0.f;
  }
  float R[9];
  rotation_from_covariance(S, R);
  float energy = 0.f;
  for (int n = 0; n < K; ++n) {
    const float s0 = valid[n] ? e0[n][0] : 0.f, s1 = valid[n] ? e0[n][1] : 0.f, s2 = valid[n] ? e0[n][2] : 0.f;
    const float d0 = (valid[n] ? et[n][0] : 0.f) - (R[0] * s0 + R[1] * s1 + R[2] * s2);
    const float d1 = (valid[n] ? et[n][1] : 0.f) - (R[3] * s0 + R[4] * s1 + R[5] * s2);
    const float d2 = (valid[n] ? et[n][2] : 0.f) - (R[6] * s0 + R[7] * s1 + R[8] * s2);
    energy += w[n] * (d0 * d0 + d1 * d1 + d2 * d2);
    const float c = 2.0f * w[n];
    g_t[n][0] = c * d0; g_t[n][1] = c * d1; g_t[n][2] = c * d2;
    g_0[n][0] = -c * (R[0] * d0 + R[3] * d1 + R[6] * d2);      // -R^T g
    g_0[n][1] = -c * (R[1] * d0 + R[4] * d1 + R[7] * d2);
    g_0[n][2] = -c * (R[2] * d0 + R[5] * d1 + R[8] * d2);
  }
  return energy;
}

}  // namespace a3d
