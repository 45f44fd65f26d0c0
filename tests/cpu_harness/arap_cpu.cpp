// CPU harness (TEST INFRASTRUCTURE) around animate3d_b200/csrc/a3d_arap_math.h: the exact __host__ __device__ edge gather and
// arithmetic of the ARAP CUDA kernels, driven serially so they can be checked against the reference goldens without a GPU.
// Build: g++ -O1 -shared -fPIC arap_cpu.cpp -o arap_cpu.so   (done by tests/test_arap_cpu.py)
#include "../../animate3d_b200/csrc/a3d_arap_math.h"

using namespace a3d;

extern "C" {

// nodes [Nt,Nv,3]; nbr [Nv,K] (-1 = absent); weight [Nv,K] or NULL (1 on existing edges); sample [Ns] node indices (entries
// outside [0, Nv) are skipped, like the kernels).  grad [Nt,Nv,3] must be zeroed.
double arap_cpu(const float* nodes, int Nt, int Nv, const int* nbr, int K, const float* weight, const int* sample, int Ns,
                float* grad) {
  double total = 0.0;
  for (int t = 1; t < Nt; ++t)
    for (int si = 0; si < Ns; ++si) {
      const int i = sample[si];
      if (i < 0 || i >= Nv) continue;             // out-of-range sample entries contribute nothing (a3d.h)
      float e0[kArapMaxK][3], et[kArapMaxK][3], g0[kArapMaxK][3], gt[kArapMaxK][3], w[kArapMaxK];
      bool valid[kArapMaxK];
      arap_gather(nodes, Nv, nbr, K, weight, i, t, e0, et, w, valid);
      total += arap_node(K, e0, et, valid, w, gt, g0);
      for (int n = 0; n < K; ++n) {
        if (!valid[n]) continue;
        const int j = nbr[i * K + n];
        for (int c = 0; c < 3; ++c) {
          grad[((long)t * Nv + i) * 3 + c] += gt[n][c];
          grad[((long)t * Nv + j) * 3 + c] -= gt[n][c];
          grad[(0 * Nv + i) * 3 + c] += g0[n][c];
          grad[(0 * Nv + j) * 3 + c] -= g0[n][c];
        }
      }
    }
  return total;
}

// rotation only (parity of R against the reference's estimate_rotation): S row-major [9] -> R row-major [9]
void arap_rotation_cpu(const float* S9, float* R9) {
  float S[3][3], R[9];
  for (int a = 0; a < 3; ++a)
    for (int b = 0; b < 3; ++b) S[a][b] = S9[a * 3 + b];
  rotation_from_covariance(S, R);
  for (int k = 0; k < 9; ++k) R9[k] = R[k];
}
}
