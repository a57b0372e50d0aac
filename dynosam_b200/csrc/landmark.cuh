// landmark.cuh -- per-landmark device helpers shared by the elimination / back-substitution kernels (kernels_schur.cu)
// and the landmark covariances (kernels_cov.cu).
#pragma once
#include "internal.cuh"

namespace dynoba {

__device__ __forceinline__ double warp_sum(double x) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
  return x;
}

// inverse of a symmetric positive definite DLxDL matrix through its Cholesky factor; false if not SPD
template <int DL>
__device__ __forceinline__ bool spd_inverse(const double* V, double* Vi) {
  if (DL == 2) {
    const double a = V[0], b = V[2], c = V[3];
    if (!(a > 0)) return false;
    const double l00 = sqrt(a), l10 = b/l00, d = c - l10*l10;
    if (!(d > 0)) return false;
    const double det = a*d;  // a*(c - b^2/a)
    Vi[0] = c/det; Vi[1] = Vi[2] = -b/det; Vi[3] = a/det;
    return true;
  } else {
    // L L^T = V
    if (!(V[0] > 0)) return false;
    const double l00 = sqrt(V[0]), l10 = V[3]/l00, l20 = V[6]/l00;
    const double d1 = V[4] - l10*l10;
    if (!(d1 > 0)) return false;
    const double l11 = sqrt(d1), l21 = (V[7] - l20*l10)/l11;
    const double d2 = V[8] - l20*l20 - l21*l21;
    if (!(d2 > 0)) return false;
    const double l22 = sqrt(d2);
    // M = L^-1 (lower)
    const double m00 = 1.0/l00, m11 = 1.0/l11, m22 = 1.0/l22;
    const double m10 = -l10*m00*m11;
    const double m21 = -l21*m11*m22;
    const double m20 = -(l20*m00 + l21*m10)*m22;
    // Vi = M^T M
    Vi[0] = m00*m00 + m10*m10 + m20*m20;
    Vi[1] = Vi[3] = m10*m11 + m20*m21;
    Vi[2] = Vi[6] = m20*m22;
    Vi[4] = m11*m11 + m21*m21;
    Vi[5] = Vi[7] = m21*m22;
    Vi[8] = m22*m22;
    return true;
  }
}

// entry (i, j) of the symmetric matrix whose lower triangle is stored in the plain band layout (tiles [NT][TPC][32x32])
__device__ __forceinline__ double band_sym(const double* __restrict__ tiles, int TPC, int i, int j) {
  if (i < j) { const int t = i; i = j; j = t; }
  return __ldg(tiles + tile_elem(TPC, j >> 5, (i >> 5) - (j >> 5), i & 31, j & 31));
}

}  // namespace dynoba
