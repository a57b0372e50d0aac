// kernels_schur.cu -- K3/K4 landmark elimination + Schur accumulation, K6 back-substitution and retraction.
//
// Restates the arithmetic GTSAM's multifrontal elimination performs on the landmark cliques
// (SURVEY.md 8a rows a11-a12; the reference's own explicit statement is
// SmartMotionFactor::createReducedMatrix / SchurComplement,
// dynosam/include/dynosam/backend/rgbd/HybridEstimator.hpp:349-396,1007-1080):
//     S   = sum_f A_f^T A_f + lambda I - W (V + lambda I)^-1 W^T,      W = A^T B, V = B^T B
//     g_S = sum_f A_f^T b_f - W (V + lambda I)^-1 g_l
// One warp owns one landmark: it stages the landmark's whitened Jacobian tiles (3x6 / 3x3, materialised by
// K1) in shared memory, reduces V and g_l with warp shuffles, inverts the 3x3 (or 2x2) block in registers and
// scatters the pairwise products  A_f^T (delta_ff' I - B_f Vinv B_f'^T) A_f'  into the tiled band storage.
#include "landmark.cuh"

namespace dynoba {

constexpr int SCHUR_WARPS = 4;

__global__ void band_clear_kernel(DevBand B) {
  const size_t stride = (size_t)gridDim.x*blockDim.x;
  double2* a = reinterpret_cast<double2*>(B.acc);           // (every buffer of the region is padded to 32 doubles)
  for (size_t i = (size_t)blockIdx.x*blockDim.x + threadIdx.x; i < B.acc_count/2; i += stride) a[i] = make_double2(0.0, 0.0);
}
// diagonal: damping lambda on the real rows, 1 on the padding rows -- written by ONE rank: rank 0 when the reduced system
// is all-reduced (world == 1 here), else the owner of the row's cell (owner(c) = c*world/ncell, as in BandPlan)
__global__ void band_diag_kernel(DevBand B, double lambda, int rank, int world) {
  const int i = blockIdx.x*blockDim.x + threadIdx.x;
  if (i >= B.n_pad) return;
  const int owner = world > 1 ? (int)((long long)band_cell(B, i)*world/B.ncell) : 0;
  if (owner != rank) return;
  *band_at(B, i, i) = i < B.n ? lambda : 1.0;
}
int launch_band_clear(const DevBand& B, double lambda, int rank, int world, cudaStream_t s) {
  band_clear_kernel<<<device_sm_count()*8, 256, 0, s>>>(B);
  band_diag_kernel<<<(B.n_pad + 255)/256, 256, 0, s>>>(B, lambda, rank, world);
  return 2;
}

// staged element accessor: element e (row-major Jacobian element, or D*JC + r for the rhs) of factor i
template <int D, int JC>
struct GroupTiles {
  const double* sJ; const DevBlock* blk; int f0; bool staged;
  __device__ __forceinline__ double operator()(int e, int i) const {
    if (staged) return sJ[e*32 + i];
    return e < D*JC ? blk->J[(size_t)e*blk->stride + f0 + i] : blk->b[(size_t)(e - D*JC)*blk->stride + f0 + i];
  }
};

template <int NP, int DL, int D, int PCOL0, int LCOL, int PSLOT0>
__global__ void __launch_bounds__(SCHUR_WARPS*32)
schur_simple_kernel(DevBlock blk, const unsigned char* __restrict__ grp_win, DevBand B, double lambda, int* __restrict__ fail) {
  constexpr int JC = NP*6 + DL, NE = D*JC + D;
  extern __shared__ double smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = blockIdx.x*SCHUR_WARPS + warp;
  if (g >= blk.n_groups || blk.grp_lmk[g] < 0 || (grp_win && grp_win[g] == 1)) return;
  double* sJ = smem + (size_t)warp*NE*32;
  const int f0 = blk.grp_ptr[g], T = blk.grp_ptr[g+1] - f0;
  const bool staged = T <= 32;
  if (staged && lane < T) {
#pragma unroll 4
    for (int e = 0; e < D*JC; e++) sJ[e*32 + lane] = blk.J[(size_t)e*blk.stride + f0 + lane];
#pragma unroll
    for (int r = 0; r < D; r++) sJ[(D*JC + r)*32 + lane] = blk.b[(size_t)r*blk.stride + f0 + lane];
  }
  __syncwarp();
  GroupTiles<D, JC> el{ sJ, &blk, f0, staged };

  // ---- pass 1: V = B^T B, g_l = B^T b (warp-shuffle reduction over the landmark's factors)
  double V[DL*DL], gl[DL];
#pragma unroll
  for (int k = 0; k < DL*DL; k++) V[k] = 0.0;
#pragma unroll
  for (int k = 0; k < DL; k++) gl[k] = 0.0;
  for (int i = lane; i < T; i += 32) {
    double Bm[D*DL], bb[D];
#pragma unroll
    for (int r = 0; r < D; r++) {
      bb[r] = el(D*JC + r, i);
#pragma unroll
      for (int c = 0; c < DL; c++) Bm[r*DL + c] = el(r*JC + LCOL + c, i);
    }
#pragma unroll
    for (int c1 = 0; c1 < DL; c1++) {
#pragma unroll
      for (int r = 0; r < D; r++) gl[c1] += Bm[r*DL + c1]*bb[r];
#pragma unroll
      for (int c2 = 0; c2 <= c1; c2++) {
#pragma unroll
        for (int r = 0; r < D; r++) V[c1*DL + c2] += Bm[r*DL + c1]*Bm[r*DL + c2];
      }
    }
  }
#pragma unroll
  for (int c1 = 0; c1 < DL; c1++) {
    gl[c1] = warp_sum(gl[c1]);
#pragma unroll
    for (int c2 = 0; c2 <= c1; c2++) { V[c1*DL + c2] = warp_sum(V[c1*DL + c2]); V[c2*DL + c1] = V[c1*DL + c2]; }
    V[c1*DL + c1] += lambda;
  }
  double Vi[DL*DL];
  if (!spd_inverse<DL>(V, Vi)) { if (lane == 0) atomicOr(fail, 1); return; }
  double vg[DL];
#pragma unroll
  for (int c = 0; c < DL; c++) { vg[c] = 0;
#pragma unroll
    for (int k = 0; k < DL; k++) vg[c] += Vi[c*DL + k]*gl[k]; }

  // ---- pass 2: g_S += A^T (b - B Vinv g_l)
  for (int i = lane; i < T; i += 32) {
    double rb[D];
#pragma unroll
    for (int r = 0; r < D; r++) {
      double s = el(D*JC + r, i);
#pragma unroll
      for (int c = 0; c < DL; c++) s -= el(r*JC + LCOL + c, i)*vg[c];
      rb[r] = s;
    }
#pragma unroll
    for (int sl = 0; sl < NP; sl++) {
      const int pos = blk.idx[(size_t)(PSLOT0 + sl)*blk.stride + f0 + i];
#pragma unroll
      for (int c = 0; c < 6; c++) {
        double a = 0;
#pragma unroll
        for (int r = 0; r < D; r++) a += el(r*JC + PCOL0 + 6*sl + c, i)*rb[r];
        red_add(rhs_at(B, pos*6 + c), a);
      }
    }
  }

  // ---- pass 3: S += A_i^T (delta_ij I - B_i Vinv B_j^T) A_j over unordered factor pairs
  const int npairs = T*(T + 1)/2;
  for (int p = lane; p < npairs; p += 32) {
    int i = (int)((sqrt(8.0*p + 1.0) - 1.0)*0.5);
    while (i*(i + 1)/2 > p) i--;
    while ((i + 1)*(i + 2)/2 <= p) i++;
    const int j = p - i*(i + 1)/2;
    double P[D*D];
    {
      double BV[D*DL];  // B_i Vinv
#pragma unroll
      for (int r = 0; r < D; r++)
#pragma unroll
        for (int c = 0; c < DL; c++) {
          double s = 0;
#pragma unroll
          for (int k = 0; k < DL; k++) s += el(r*JC + LCOL + k, i)*Vi[k*DL + c];
          BV[r*DL + c] = s;
        }
#pragma unroll
      for (int r = 0; r < D; r++)
#pragma unroll
        for (int q = 0; q < D; q++) {
          double s = (i == j && r == q) ? 1.0 : 0.0;
#pragma unroll
          for (int c = 0; c < DL; c++) s -= BV[r*DL + c]*el(q*JC + LCOL + c, j);
          P[r*D + q] = s;
        }
    }
#pragma unroll
    for (int s1 = 0; s1 < NP; s1++) {
      const int a = blk.idx[(size_t)(PSLOT0 + s1)*blk.stride + f0 + i];
      double Ai[D*6];
#pragma unroll
      for (int r = 0; r < D; r++)
#pragma unroll
        for (int c = 0; c < 6; c++) Ai[r*6 + c] = el(r*JC + PCOL0 + 6*s1 + c, i);
#pragma unroll
      for (int s2 = 0; s2 < NP; s2++) {
        if (i == j && s2 > s1) continue;
        const int b = blk.idx[(size_t)(PSLOT0 + s2)*blk.stride + f0 + j];
        double PA[D*6];
#pragma unroll
        for (int r = 0; r < D; r++)
#pragma unroll
          for (int c = 0; c < 6; c++) {
            double s = 0;
#pragma unroll
            for (int q = 0; q < D; q++) s += P[r*D + q]*el(q*JC + PCOL0 + 6*s2 + c, j);
            PA[r*6 + c] = s;
          }
        const bool same = (i == j && s1 == s2);
        const BandBlockRef cref = band_block_ref(B, (a > b ? a : b)*6, (a < b ? a : b)*6);   // the block's storage, resolved once
#pragma unroll
        for (int c = 0; c < 6; c++) {
#pragma unroll
          for (int c2 = 0; c2 < 6; c2++) {
            if (same && c2 > c) continue;
            double m = 0;
#pragma unroll
            for (int r = 0; r < D; r++) m += Ai[r*6 + c]*PA[r*6 + c2];
            const int row = a*6 + c, col = b*6 + c2;
            if (a > b || same) red_add(band_block_at(B, cref, row, col), m);
            else if (a < b) red_add(band_block_at(B, cref, col, row), m);
            else {  // two different factor slots on the same variable: contributes M + M^T
              const int hi = row > col ? row : col, lo = row > col ? col : row;
              red_add(band_block_at(B, cref, hi, lo), c == c2 ? 2.0*m : m);
            }
          }
        }
      }
    }
  }
}

template <int NP, int DL, int D, int PCOL0, int LCOL, int PSLOT0>
static int launch_schur_t(const DevBlock& blk, const unsigned char* grp_win, const DevBand& B, double lambda, int* fail, cudaStream_t s) {
  constexpr int NE = D*(NP*6 + DL) + D;
  const size_t smem = (size_t)SCHUR_WARPS*NE*32*sizeof(double);
  auto kern = schur_simple_kernel<NP, DL, D, PCOL0, LCOL, PSLOT0>;
  static bool attr_set = false;
  if (!attr_set) { cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem); attr_set = true; }
  const int grid = (blk.n_groups + SCHUR_WARPS - 1)/SCHUR_WARPS;
  kern<<<grid, SCHUR_WARPS*32, smem, s>>>(blk, grp_win, B, lambda, fail);
  return 1;
}

int launch_schur_simple(const DevBlock& blk, const unsigned char* grp_win, const DevBand& B, double lambda, int* fail, cudaStream_t s) {
  if (blk.n_groups == 0) return 0;
  switch (blk.type) {
    case F_POSE2POINT3: case F_STEREO3: case F_LINEAR_PP3: return launch_schur_t<1, 3, 3, 0, 6, 0>(blk, grp_win, B, lambda, fail, s);
    case F_HYBRID3: case F_HYBRID_STEREO3: case F_LINEAR_PPP3: return launch_schur_t<2, 3, 3, 0, 12, 0>(blk, grp_win, B, lambda, fail, s);
    case F_FLOWPROJ2: return launch_schur_t<1, 2, 2, 2, 0, 1>(blk, grp_win, B, lambda, fail, s);
    default: return 0;
  }
}

// ---- pose-only factors (PRIOR6, BETWEEN6, SMOOTH_*): J^T J and J^T b straight into S / g_S
__global__ void pose_factors_kernel(DevBlock blk, DevBand B, int arity) {
  const int f = blockIdx.x*blockDim.x + threadIdx.x;
  if (f >= blk.n) return;
  const int JC = 6*arity;
  double bb[6];
#pragma unroll
  for (int r = 0; r < 6; r++) bb[r] = blk.b[(size_t)r*blk.stride + f];
  for (int k1 = 0; k1 < arity; k1++) {
    const int a = blk.idx[(size_t)k1*blk.stride + f];
    for (int c = 0; c < 6; c++) {
      double g = 0;
#pragma unroll
      for (int r = 0; r < 6; r++) g += blk.J[(size_t)(r*JC + 6*k1 + c)*blk.stride + f]*bb[r];
      red_add(rhs_at(B, a*6 + c), g);
    }
    for (int k2 = 0; k2 <= k1; k2++) {
      const int b = blk.idx[(size_t)k2*blk.stride + f];
        const BandBlockRef cref = band_block_ref(B, (a > b ? a : b)*6, (a < b ? a : b)*6);   // the block's storage, resolved once
      for (int c = 0; c < 6; c++)
        for (int c2 = 0; c2 < 6; c2++) {
          if (k1 == k2 && c2 > c) continue;
          double m = 0;
#pragma unroll
          for (int r = 0; r < 6; r++)
            m += blk.J[(size_t)(r*JC + 6*k1 + c)*blk.stride + f]*blk.J[(size_t)(r*JC + 6*k2 + c2)*blk.stride + f];
          const int row = a*6 + c, col = b*6 + c2;
          if (a > b || k1 == k2) red_add(band_block_at(B, cref, row, col), m);
          else if (a < b) red_add(band_block_at(B, cref, col, row), m);
          else { const int hi = row > col ? row : col, lo = row > col ? col : row;
                 red_add(band_block_at(B, cref, hi, lo), c == c2 ? 2.0*m : m); }
        }
    }
  }
}
int launch_pose_factors(const DevBlock& blk, const DevBand& B, cudaStream_t s) {
  if (blk.n == 0) return 0;
  if (is_nav_type(blk.type)) return launch_nav_factors(blk, B, s);
  pose_factors_kernel<<<(blk.n + 127)/128, 128, 0, s>>>(blk, B, type_info(blk.type).arity);
  return 1;
}

// ---- K6: back-substitution  delta_l = Vinv (g_l - W^T delta_p)  + model-decrease partial sums
template <int NP, int DL, int D, int PCOL0, int LCOL, int PSLOT0>
__global__ void __launch_bounds__(SCHUR_WARPS*32)
backsub_simple_kernel(DevBlock blk, DevBand B, double lambda, double* __restrict__ dl, int dl_stride,
                      double* __restrict__ partials) {
  constexpr int JC = NP*6 + DL;
  __shared__ double sh[SCHUR_WARPS];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = blockIdx.x*SCHUR_WARPS + warp;
  double model = 0.0;
  if (g < blk.n_groups && blk.grp_lmk[g] >= 0) {
    const int f0 = blk.grp_ptr[g], T = blk.grp_ptr[g+1] - f0;
    double V[DL*DL], gl[DL], tw[DL], q1 = 0.0;
#pragma unroll
    for (int k = 0; k < DL*DL; k++) V[k] = 0.0;
#pragma unroll
    for (int k = 0; k < DL; k++) { gl[k] = 0.0; tw[k] = 0.0; }
    for (int i = lane; i < T; i += 32) {
      const int f = f0 + i;
      double Bm[D*DL], bb[D], u[D];
#pragma unroll
      for (int r = 0; r < D; r++) {
        bb[r] = blk.b[(size_t)r*blk.stride + f]; u[r] = 0.0;
#pragma unroll
        for (int c = 0; c < DL; c++) Bm[r*DL + c] = blk.J[(size_t)(r*JC + LCOL + c)*blk.stride + f];
      }
#pragma unroll
      for (int sl = 0; sl < NP; sl++) {
        const int pos = blk.idx[(size_t)(PSLOT0 + sl)*blk.stride + f];
        double dp[6];
#pragma unroll
        for (int c = 0; c < 6; c++) dp[c] = B.dp[pos*6 + c];
#pragma unroll
        for (int r = 0; r < D; r++)
#pragma unroll
          for (int c = 0; c < 6; c++) u[r] += blk.J[(size_t)(r*JC + PCOL0 + 6*sl + c)*blk.stride + f]*dp[c];
      }
#pragma unroll
      for (int r = 0; r < D; r++) q1 += bb[r]*u[r];
#pragma unroll
      for (int c1 = 0; c1 < DL; c1++) {
#pragma unroll
        for (int r = 0; r < D; r++) { gl[c1] += Bm[r*DL + c1]*bb[r]; tw[c1] += Bm[r*DL + c1]*u[r]; }
#pragma unroll
        for (int c2 = 0; c2 <= c1; c2++)
#pragma unroll
          for (int r = 0; r < D; r++) V[c1*DL + c2] += Bm[r*DL + c1]*Bm[r*DL + c2];
      }
    }
    q1 = warp_sum(q1);
#pragma unroll
    for (int c1 = 0; c1 < DL; c1++) {
      gl[c1] = warp_sum(gl[c1]); tw[c1] = warp_sum(tw[c1]);
#pragma unroll
      for (int c2 = 0; c2 <= c1; c2++) { V[c1*DL + c2] = warp_sum(V[c1*DL + c2]); V[c2*DL + c1] = V[c1*DL + c2]; }
      V[c1*DL + c1] += lambda;
    }
    double Vi[DL*DL];
    if (spd_inverse<DL>(V, Vi)) {
      double d[DL], gd = 0, dd = 0;
#pragma unroll
      for (int c = 0; c < DL; c++) {
        double s = 0;
#pragma unroll
        for (int k = 0; k < DL; k++) s += Vi[c*DL + k]*(gl[k] - tw[k]);
        d[c] = s; gd += gl[c]*s; dd += s*s;
      }
      if (lane == 0) {
        const int l = blk.grp_lmk[g];
#pragma unroll
        for (int c = 0; c < DL; c++) dl[(size_t)c*dl_stride + l] = d[c];
      }
      model = 0.5*(q1 + gd) + 0.5*lambda*dd;
    }
  }
  if (lane == 0) sh[warp] = model;
  __syncthreads();
  if (threadIdx.x == 0) { double t = 0; for (int w = 0; w < SCHUR_WARPS; w++) t += sh[w]; partials[blockIdx.x] = t; }
}

int backsub_grid(int n_groups) { return (n_groups + SCHUR_WARPS - 1)/SCHUR_WARPS; }

int launch_backsub_simple(const DevBlock& blk, const DevBand& B, double lambda, double* dl_point, int nl_stride,
                          double* dl_flow, int nf_stride, double* partials, cudaStream_t s) {
  if (blk.n_groups == 0) return 0;
  const int grid = backsub_grid(blk.n_groups);
  switch (blk.type) {
    case F_POSE2POINT3: case F_STEREO3: case F_LINEAR_PP3:
      backsub_simple_kernel<1, 3, 3, 0, 6, 0><<<grid, SCHUR_WARPS*32, 0, s>>>(blk, B, lambda, dl_point, nl_stride, partials); return 1;
    case F_HYBRID3: case F_HYBRID_STEREO3: case F_LINEAR_PPP3:
      backsub_simple_kernel<2, 3, 3, 0, 12, 0><<<grid, SCHUR_WARPS*32, 0, s>>>(blk, B, lambda, dl_point, nl_stride, partials); return 1;
    case F_FLOWPROJ2:
      backsub_simple_kernel<1, 2, 2, 2, 0, 1><<<grid, SCHUR_WARPS*32, 0, s>>>(blk, B, lambda, dl_flow, nf_stride, partials); return 1;
    default: return 0;
  }
}

// pose-only factors' share of g^T delta:  0.5 * b^T (A delta_p)
__global__ void pose_model_kernel(DevBlock blk, DevBand B, int arity, double* __restrict__ partials) {
  __shared__ double sh[128];
  const int f = blockIdx.x*blockDim.x + threadIdx.x;
  double q = 0;
  if (f < blk.n) {
    const int JC = 6*arity;
    for (int r = 0; r < 6; r++) {
      double u = 0;
      for (int k = 0; k < arity; k++) {
        const int a = blk.idx[(size_t)k*blk.stride + f];
        for (int c = 0; c < 6; c++) u += blk.J[(size_t)(r*JC + 6*k + c)*blk.stride + f]*B.dp[a*6 + c];
      }
      q += blk.b[(size_t)r*blk.stride + f]*u;
    }
    q *= 0.5;
  }
  sh[threadIdx.x] = q;
  __syncthreads();
  for (int o = 64; o > 0; o >>= 1) { if ((int)threadIdx.x < o) sh[threadIdx.x] += sh[threadIdx.x + o]; __syncthreads(); }
  if (threadIdx.x == 0) partials[blockIdx.x] = sh[0];
}
int launch_pose_model(const DevBlock& blk, const DevBand& B, double* partials, cudaStream_t s) {
  if (blk.n == 0) return 0;
  if (is_nav_type(blk.type)) return launch_nav_model(blk, B, partials, s);
  pose_model_kernel<<<(blk.n + 127)/128, 128, 0, s>>>(blk, B, type_info(blk.type).arity, partials);
  return 1;
}

__global__ void pose_delta_norm_kernel(DevBand B, double lambda, double* __restrict__ partials) {
  __shared__ double sh[256];
  const int i = blockIdx.x*blockDim.x + threadIdx.x;
  double q = 0;
  if (i < B.n) { const double d = B.dp[i]; q = 0.5*lambda*d*d; }
  sh[threadIdx.x] = q;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) { if ((int)threadIdx.x < o) sh[threadIdx.x] += sh[threadIdx.x + o]; __syncthreads(); }
  if (threadIdx.x == 0) partials[blockIdx.x] = sh[0];
}
int pose_norm_grid(int n) { return (n + 255)/256; }
int launch_pose_delta_norm(const DevBand& B, double lambda, double* partials, cudaStream_t s) {
  pose_delta_norm_kernel<<<pose_norm_grid(B.n), 256, 0, s>>>(B, lambda, partials);
  return 1;
}

// ---- values.retract(delta): Pose3 -> T * Expmap(xi), Point3 / flow -> p + d
__global__ void retract_pose_kernel(DevVars cur, DevVars cand, const double* __restrict__ dp) {
  const int p = blockIdx.x*blockDim.x + threadIdx.x;
  if (p >= cur.np) return;
  Pose P, O;
#pragma unroll
  for (int k = 0; k < 9; k++) P.R[k] = cur.pose[(size_t)k*cur.np_stride + p];
#pragma unroll
  for (int k = 0; k < 3; k++) P.t[k] = cur.pose[(size_t)(9 + k)*cur.np_stride + p];
  double xi[6];
#pragma unroll
  for (int c = 0; c < 6; c++) xi[c] = dp[p*6 + c];
  se3_retract(P, xi, O);
#pragma unroll
  for (int k = 0; k < 9; k++) cand.pose[(size_t)k*cand.np_stride + p] = O.R[k];
#pragma unroll
  for (int k = 0; k < 3; k++) cand.pose[(size_t)(9 + k)*cand.np_stride + p] = O.t[k];
}
__global__ void retract_vec_kernel(const double* __restrict__ cur, double* __restrict__ cand, const double* __restrict__ d, size_t n) {
  const size_t i = (size_t)blockIdx.x*blockDim.x + threadIdx.x;
  if (i < n) cand[i] = cur[i] + d[i];
}
int launch_retract(const DevVars& cur, const DevVars& cand, const DevBand& B, const double* dl_point,
                   const double* dl_flow, cudaStream_t s) {
  int k = 0;
  if (cur.np) { retract_pose_kernel<<<(cur.np + 127)/128, 128, 0, s>>>(cur, cand, B.dp); k++; }
  if (cur.nl) { const size_t n = (size_t)3*cur.nl_stride; retract_vec_kernel<<<(unsigned)((n + 255)/256), 256, 0, s>>>(cur.point, cand.point, dl_point, n); k++; }
  if (cur.nf) { const size_t n = (size_t)2*cur.nf_stride; retract_vec_kernel<<<(unsigned)((n + 255)/256), 256, 0, s>>>(cur.flow, cand.flow, dl_flow, n); k++; }
  return k;
}

}  // namespace dynoba
