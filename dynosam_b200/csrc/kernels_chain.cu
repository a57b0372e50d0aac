// kernels_chain.cu -- landmark elimination for GENERAL landmark groups: several point variables chained by
// LandmarkMotionTernaryFactor (WCME, dynosam/src/backend/rgbd/WorldMotionEstimator.cc:151-274) or
// LandmarkMotionPoseFactor (WCPE, src/backend/rgbd/WorldPoseEstimator.cc:89-315), or a single point whose
// factors live in more than one factor block.  The landmark block V of such a group is block-tridiagonal
// (SURVEY.md section 7 "hard parts"); with at most 21 points per tracklet it is handled densely:
// one warp per group builds V (<= 63x63) in shared memory, inverts it through its Cholesky factor and scatters
//   S += A_f^T (delta_ff' I - B_f Vinv[lm(f), lm(f')] B_f'^T) A_f'   over the group's factor pairs.
#include "landmark.cuh"

namespace dynoba {

constexpr int GG_MAXL = 21;            // points per group
constexpr int GG_N = 3*GG_MAXL;        // 63
constexpr int GG_LD = GG_N + 1;        // padded leading dimension

struct FRef { int blk, idx; };

// runtime view of one factor's linearisation (all landmark factors have D = 3 rows here)
struct FView {
  const DevBlock* b; int f, jc, np, nl; int pcol[2], lcol[2], pslot[2], lslot[2];
  __device__ __forceinline__ double J(int r, int c) const { return b->J[(size_t)(r*jc + c)*b->stride + f]; }
  __device__ __forceinline__ double rhs(int r) const { return b->b[(size_t)r*b->stride + f]; }
  __device__ __forceinline__ int pose(int s) const { return b->idx[(size_t)pslot[s]*b->stride + f]; }
  __device__ __forceinline__ int lmk(int s) const { return b->idx[(size_t)lslot[s]*b->stride + f]; }
};
__device__ __forceinline__ FView make_view(const DevBlock* blocks, FRef r) {
  FView v; v.b = blocks + r.blk; v.f = r.idx;
  const TypeInfo ti = type_info(v.b->type);
  v.jc = ti.jcols; v.np = 0; v.nl = 0;
  for (int k = 0; k < ti.arity; k++) {
    if (ti.cls[k] == VC_POSE) { v.pcol[v.np] = ti.coloff[k]; v.pslot[v.np] = k; v.np++; }
    else { v.lcol[v.nl] = ti.coloff[k]; v.lslot[v.nl] = k; v.nl++; }
  }
  return v;
}

// builds V + lambda I and g_l in shared memory, replaces V by its inverse; returns false if not SPD
__device__ bool group_inverse(const DevBlock* blocks, const FRef* refs, int nf, int l0, int n, double lambda,
                              double* V, double* gl, double* W, int lane) {
  for (int i = lane; i < n*GG_LD; i += 32) V[i] = 0.0;
  for (int i = lane; i < n; i += 32) gl[i] = 0.0;
  __syncwarp();
  for (int q = 0; q < nf; q++) {      // factors serially, lanes over the entries of the factor's local Hessian
    const FView v = make_view(blocks, refs[q]);
    const int nloc = 3*v.nl;
    for (int e = lane; e < nloc*nloc + nloc; e += 32) {
      if (e < nloc*nloc) {
        const int i = e/nloc, j = e%nloc;
        const int gi = 3*(v.lmk(i/3) - l0) + i%3, gj = 3*(v.lmk(j/3) - l0) + j%3;
        double s = 0;
        for (int r = 0; r < 3; r++) s += v.J(r, v.lcol[i/3] + i%3)*v.J(r, v.lcol[j/3] + j%3);
        V[gi*GG_LD + gj] += s;
      } else {
        const int i = e - nloc*nloc;
        const int gi = 3*(v.lmk(i/3) - l0) + i%3;
        double s = 0;
        for (int r = 0; r < 3; r++) s += v.J(r, v.lcol[i/3] + i%3)*v.rhs(r);
        gl[gi] += s;
      }
    }
    __syncwarp();
  }
  for (int i = lane; i < n; i += 32) V[i*GG_LD + i] += lambda;
  __syncwarp();
  // Cholesky (lower, in place), column by column
  bool ok = true;
  for (int k = 0; k < n; k++) {
    const double d = V[k*GG_LD + k];
    if (!(d > 0.0)) { ok = false; break; }
    const double inv = rsqrt(d);
    __syncwarp();
    for (int i = k + lane; i < n; i += 32) V[i*GG_LD + k] = (i == k) ? d*inv : V[i*GG_LD + k]*inv;
    __syncwarp();
    for (int i = k + 1 + lane; i < n; i += 32) {
      const double lik = V[i*GG_LD + k];
      for (int j = k + 1; j <= i; j++) V[i*GG_LD + j] -= lik*V[j*GG_LD + k];
    }
    __syncwarp();
  }
  if (!ok) return false;
  // W = L^-1 (lower): column j solved by lane j%32
  for (int j = lane; j < n; j += 32) {
    for (int i = 0; i < n; i++) {
      double s = (i == j) ? 1.0 : 0.0;
      for (int k = j; k < i; k++) s -= V[i*GG_LD + k]*W[k*GG_LD + j];
      W[i*GG_LD + j] = (i >= j) ? s/V[i*GG_LD + i] : 0.0;
    }
  }
  __syncwarp();
  // Vinv = W^T W (symmetric), written over V
  for (int e = lane; e < n*n; e += 32) {
    const int i = e/n, j = e%n;
    if (j > i) continue;
    double s = 0;
    for (int k = i; k < n; k++) s += W[k*GG_LD + i]*W[k*GG_LD + j];
    V[i*GG_LD + j] = s; V[j*GG_LD + i] = s;
  }
  __syncwarp();
  return true;
}

// P = delta I - sum_{s,s'} B_{f,s} Vinv[l_s, l_s'] B_{f',s'}^T   (3x3)
__device__ __forceinline__ void pair_projector(const FView& a, const FView& b, bool same, int l0, const double* Vi, double* P) {
  for (int e = 0; e < 9; e++) P[e] = (same && e%4 == 0) ? 1.0 : 0.0;
  for (int s = 0; s < a.nl; s++) for (int t = 0; t < b.nl; t++) {
    const int oa = 3*(a.lmk(s) - l0), ob = 3*(b.lmk(t) - l0);
    double BV[9];
    for (int r = 0; r < 3; r++) for (int c = 0; c < 3; c++) {
      double x = 0;
      for (int k = 0; k < 3; k++) x += a.J(r, a.lcol[s] + k)*Vi[(oa + k)*GG_LD + ob + c];
      BV[3*r + c] = x;
    }
    for (int r = 0; r < 3; r++) for (int q = 0; q < 3; q++) {
      double x = 0;
      for (int c = 0; c < 3; c++) x += BV[3*r + c]*b.J(q, b.lcol[t] + c);
      P[3*r + q] -= x;
    }
  }
}

__global__ void __launch_bounds__(64)
schur_general_kernel(const DevBlock* __restrict__ blocks, const int* __restrict__ gptr, const FRef* __restrict__ refs,
                     const int* __restrict__ gl0, const int* __restrict__ gnl, int n_groups, DevBand B, double lambda,
                     int* __restrict__ fail) {
  extern __shared__ double sm[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = blockIdx.x*2 + warp;
  if (g >= n_groups) return;
  double* V = sm + (size_t)warp*(2*GG_N*GG_LD + GG_N);
  double* W = V + GG_N*GG_LD; double* gl = W + GG_N*GG_LD;
  const int f0 = gptr[g], nf = gptr[g+1] - f0, l0 = gl0[g], n = 3*gnl[g];
  const FRef* rf = refs + f0;
  if (!group_inverse(blocks, rf, nf, l0, n, lambda, V, gl, W, lane)) { if (lane == 0) atomicOr(fail, 1); return; }
  // vg = Vinv g_l (into W row 0)
  double* vg = W;
  for (int i = lane; i < n; i += 32) { double s = 0; for (int k = 0; k < n; k++) s += V[i*GG_LD + k]*gl[k]; vg[i] = s; }
  __syncwarp();
  // gradient
  for (int q = lane; q < nf; q += 32) {
    const FView v = make_view(blocks, rf[q]);
    double rb[3];
    for (int r = 0; r < 3; r++) {
      double s = v.rhs(r);
      for (int t = 0; t < v.nl; t++) for (int c = 0; c < 3; c++) s -= v.J(r, v.lcol[t] + c)*vg[3*(v.lmk(t) - l0) + c];
      rb[r] = s;
    }
    for (int s = 0; s < v.np; s++) {
      const int pos = v.pose(s);
      for (int c = 0; c < 6; c++) { double a = 0; for (int r = 0; r < 3; r++) a += v.J(r, v.pcol[s] + c)*rb[r]; red_add(rhs_at(B, pos*6 + c), a); }
    }
  }
  // factor pairs
  const int npairs = nf*(nf + 1)/2;
  for (int p = lane; p < npairs; p += 32) {
    int i = (int)((sqrt(8.0*p + 1.0) - 1.0)*0.5);
    while (i*(i + 1)/2 > p) i--;
    while ((i + 1)*(i + 2)/2 <= p) i++;
    const int j = p - i*(i + 1)/2;
    const FView vi = make_view(blocks, rf[i]), vj = make_view(blocks, rf[j]);
    double P[9];
    pair_projector(vi, vj, i == j, l0, V, P);
    for (int s1 = 0; s1 < vi.np; s1++) {
      const int a = vi.pose(s1);
      for (int s2 = 0; s2 < vj.np; s2++) {
        if (i == j && s2 > s1) continue;
        const int b = vj.pose(s2);
        const bool same = (i == j && s1 == s2);
        double PA[18];
        for (int r = 0; r < 3; r++) for (int c = 0; c < 6; c++) {
          double s = 0; for (int q = 0; q < 3; q++) s += P[3*r + q]*vj.J(q, vj.pcol[s2] + c);
          PA[6*r + c] = s;
        }
        const BandBlockRef cref = band_block_ref(B, (a > b ? a : b)*6, (a < b ? a : b)*6);   // the block's storage, resolved once
        for (int c = 0; c < 6; c++) {
          double ai[3]; for (int r = 0; r < 3; r++) ai[r] = vi.J(r, vi.pcol[s1] + c);
          for (int c2 = 0; c2 < 6; c2++) {
            if (same && c2 > c) continue;
            const double m = ai[0]*PA[c2] + ai[1]*PA[6 + c2] + ai[2]*PA[12 + c2];
            const int row = a*6 + c, col = b*6 + c2;
            if (a > b || same) red_add(band_block_at(B, cref, row, col), m);
            else if (a < b) red_add(band_block_at(B, cref, col, row), m);
            else { const int hi = row > col ? row : col, lo = row > col ? col : row;
                   red_add(band_block_at(B, cref, hi, lo), c == c2 ? 2.0*m : m); }
          }
        }
      }
    }
  }
}

__global__ void __launch_bounds__(64)
backsub_general_kernel(const DevBlock* __restrict__ blocks, const int* __restrict__ gptr, const FRef* __restrict__ refs,
                       const int* __restrict__ gl0, const int* __restrict__ gnl, int n_groups, DevBand B, double lambda,
                       double* __restrict__ dl, int dl_stride, double* __restrict__ partials) {
  extern __shared__ double sm[];
  __shared__ double sh[2];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = blockIdx.x*2 + warp;
  double model = 0.0;
  if (g < n_groups) {
    double* V = sm + (size_t)warp*(2*GG_N*GG_LD + 2*GG_N);
    double* W = V + GG_N*GG_LD; double* gl = W + GG_N*GG_LD; double* tw = gl + GG_N;
    const int f0 = gptr[g], nf = gptr[g+1] - f0, l0 = gl0[g], n = 3*gnl[g];
    const FRef* rf = refs + f0;
    if (group_inverse(blocks, rf, nf, l0, n, lambda, V, gl, W, lane)) {
      for (int i = lane; i < n; i += 32) tw[i] = 0.0;
      __syncwarp();
      double q1 = 0;
      for (int q = 0; q < nf; q++) {     // serial over factors: several factors add to the same landmark
        const FView v = make_view(blocks, rf[q]);
        double u[3] = {0, 0, 0};
        for (int s = 0; s < v.np; s++) { const int pos = v.pose(s);
          for (int r = 0; r < 3; r++) for (int c = 0; c < 6; c++) u[r] += v.J(r, v.pcol[s] + c)*B.dp[pos*6 + c]; }
        if (lane == 0) for (int r = 0; r < 3; r++) q1 += v.rhs(r)*u[r];
        if (lane < 3*v.nl) {
          const int t = lane/3, c = lane%3;
          double s = 0; for (int r = 0; r < 3; r++) s += v.J(r, v.lcol[t] + c)*u[r];
          tw[3*(v.lmk(t) - l0) + c] += s;
        }
        __syncwarp();
      }
      double gd = 0, dd = 0;
      for (int i = lane; i < n; i += 32) {
        double s = 0; for (int k = 0; k < n; k++) s += V[i*GG_LD + k]*(gl[k] - tw[k]);
        dl[(size_t)(i%3)*dl_stride + l0 + i/3] = s;
        gd += gl[i]*s; dd += s*s;
      }
      for (int o = 16; o > 0; o >>= 1) { gd += __shfl_xor_sync(0xffffffffu, gd, o); dd += __shfl_xor_sync(0xffffffffu, dd, o); }
      q1 = __shfl_sync(0xffffffffu, q1, 0);
      model = 0.5*(q1 + gd) + 0.5*lambda*dd;
    }
  }
  if (lane == 0) sh[warp] = model;
  __syncthreads();
  if (threadIdx.x == 0) partials[blockIdx.x] = sh[0] + sh[1];
}

// Marginal covariances of a general group's points (dynoba_marginal_covariance; here because it shares
// group_inverse): with V^-1 the group's dense undamped inverse and Y = W^T Sigma_cc W summed over the pairs of
// (factor, pose slot) terms, Sigma_points = V^-1 + V^-1 Y V^-1, of which each point's 3x3 diagonal block is kept.
__global__ void __launch_bounds__(64)
cov_general_kernel(const DevBlock* __restrict__ blocks, const int* __restrict__ gptr, const FRef* __restrict__ refs,
                   const int* __restrict__ gl0, const int* __restrict__ gnl, int n_groups, const double* __restrict__ sig,
                   int TPC, double* __restrict__ out, int* __restrict__ fail) {
  extern __shared__ double sm[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = blockIdx.x*2 + warp;
  if (g >= n_groups) return;
  double* V = sm + (size_t)warp*(2*GG_N*GG_LD + 2*GG_N);
  double* W = V + GG_N*GG_LD; double* gl = W + GG_N*GG_LD;
  const int f0 = gptr[g], nf = gptr[g+1] - f0, l0 = gl0[g], nl = gnl[g], n = 3*nl;
  const FRef* rf = refs + f0;
  if (!group_inverse(blocks, rf, nf, l0, n, 0.0, V, gl, W, lane)) { if (lane == 0) atomicOr(fail, 1); return; }
  double* Y = W;
  for (int i = lane; i < n*GG_LD; i += 32) Y[i] = 0.0;
  __syncwarp();
  for (int p = lane; p < nf*nf; p += 32) {
    const FView a = make_view(blocks, rf[p/nf]), b = make_view(blocks, rf[p%nf]);
    for (int s1 = 0; s1 < a.np; s1++) for (int s2 = 0; s2 < b.np; s2++) {
      const int pa = 6*a.pose(s1), pb = 6*b.pose(s2);
      double Sg[36];
      for (int c = 0; c < 6; c++) for (int c2 = 0; c2 < 6; c2++) Sg[c*6 + c2] = band_sym(sig, TPC, pa + c, pb + c2);
      for (int t1 = 0; t1 < a.nl; t1++) {
        double G[18];                                   // (B_a,t1^T A_a,s1) Sigma(pa, pb)
        for (int k = 0; k < 3; k++) {
          double ca[6];
          for (int c = 0; c < 6; c++) { double x = 0; for (int r = 0; r < 3; r++) x += a.J(r, a.lcol[t1] + k)*a.J(r, a.pcol[s1] + c); ca[c] = x; }
          for (int c2 = 0; c2 < 6; c2++) { double x = 0; for (int c = 0; c < 6; c++) x += ca[c]*Sg[c*6 + c2]; G[k*6 + c2] = x; }
        }
        for (int t2 = 0; t2 < b.nl; t2++) {
          for (int k2 = 0; k2 < 3; k2++) {
            double cb[6];
            for (int c = 0; c < 6; c++) { double x = 0; for (int r = 0; r < 3; r++) x += b.J(r, b.lcol[t2] + k2)*b.J(r, b.pcol[s2] + c); cb[c] = x; }
            for (int k = 0; k < 3; k++) {
              double x = 0; for (int c = 0; c < 6; c++) x += G[k*6 + c]*cb[c];
              atomicAdd(Y + (3*(a.lmk(t1) - l0) + k)*GG_LD + 3*(b.lmk(t2) - l0) + k2, x);
            }
          }
        }
      }
    }
  }
  __syncwarp();
  for (int e = lane; e < 6*nl; e += 32) {               // lower entries (r >= c) of each point's block
    const int l = e/6, q = e%6, r = q < 1 ? 0 : (q < 3 ? 1 : 2), c = q - r*(r + 1)/2;
    const int ir = 3*l + r, ic = 3*l + c;
    double s = V[ir*GG_LD + ic];
    for (int i = 0; i < n; i++) {
      double t = 0;
      for (int k = 0; k < n; k++) t += Y[i*GG_LD + k]*V[k*GG_LD + ic];
      s += V[ir*GG_LD + i]*t;
    }
    double* o = out + (size_t)(l0 + l)*9;
    o[r*3 + c] = s; o[c*3 + r] = s;
  }
}

static size_t gg_smem() { return (size_t)2*(2*GG_N*GG_LD + 2*GG_N)*sizeof(double); }

// Requested-landmark strips of dynoba_joint_marginal_covariance (here because it shares group_inverse), one warp per
// requested landmark group g (a point alone, a WCME / WCPE chain, or a flow).  With V_g^-1 the group's undamped inverse
// and W the pose-landmark block of H, for every requested landmark l of the group:
//     M_l = (W V_g^-1)[C, l]   = sum over the (factor, pose slot) terms b of U_b^T (V_g^-1)[., l],  U_b = B_f^T A_{f,s}
//     Z_l = Sigma(l, C)        = -M_l^T X[C, C]    (= -V_g^-1 W^T S^-1 restricted to C: every pose of W[., g] is in C)
// and V_g^-1 itself; the host then forms Sigma(l1, l2) = delta_g (V_g^-1)(l1, l2) - Z_l1 M_l2.
static_assert(STRIP_LD == GG_N, "a group's V^-1 is returned with the leading dimension of the largest group");
__global__ void __launch_bounds__(64) cov_strip_kernel(StripJob j) {
  extern __shared__ double sm[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = blockIdx.x*2 + warp;
  if (g >= j.ng) return;
  double* V = sm + (size_t)warp*(2*GG_N*GG_LD + 2*GG_N);
  double* W = V + GG_N*GG_LD; double* gl = W + GG_N*GG_LD;
  const int4 G = j.groups[g];
  const FRef* rf = (const FRef*)j.refs + G.x;
  const int nf = G.y - G.x, l0 = G.z;
  const bool flow = G.w == 0;
  const int ld = flow ? 2 : 3, rows = flow ? 2 : 3, n = flow ? 2 : 3*G.w;
  if (flow) {                 // one flow: V = sum_f B_f^T B_f (2x2)
    double v[4] = {0.0, 0.0, 0.0, 0.0};
    for (int q = lane; q < nf; q += 32) {
      const FView f = make_view(j.blocks, rf[q]);
      for (int r = 0; r < 2; r++) { const double b0 = f.J(r, f.lcol[0]), b1 = f.J(r, f.lcol[0] + 1); v[0] += b0*b0; v[1] += b0*b1; v[3] += b1*b1; }
    }
    for (int e = 0; e < 4; e++) v[e] = warp_sum(v[e]);
    v[2] = v[1];
    double vi[4];
    if (!spd_inverse<2>(v, vi)) { if (lane == 0) atomicOr(j.fail, 1); return; }
    if (lane == 0) { V[0] = vi[0]; V[1] = vi[1]; V[GG_LD] = vi[2]; V[GG_LD + 1] = vi[3]; }
    __syncwarp();
  } else if (!group_inverse(j.blocks, rf, nf, l0, n, 0.0, V, gl, W, lane)) { if (lane == 0) atomicOr(j.fail, 1); return; }
  for (int e = lane; e < n*n; e += 32) j.vinv[(size_t)g*STRIP_LD*STRIP_LD + (size_t)(e/n)*STRIP_LD + e%n] = V[(e/n)*GG_LD + e%n];
  for (int q = j.rptr[g]; q < j.rptr[g + 1]; q++) {
    const int o = ld*(j.rl[q] - l0);
    double* mq = j.m + (size_t)q*j.nc*3;
    for (int p = lane; p < 2*nf; p += 32) {   // terms (factor p/2, pose slot p%2) over the lanes
      const FView f = make_view(j.blocks, rf[p >> 1]);
      const int s = p & 1;
      if (s >= f.np) continue;
      const int c0 = j.cmap[f.pose(s)];
      double acc[6][3];
#pragma unroll
      for (int c = 0; c < 6; c++)
#pragma unroll
        for (int k = 0; k < 3; k++) acc[c][k] = 0.0;
      for (int t = 0; t < f.nl; t++) {
        const int ot = ld*(f.lmk(t) - l0);
        for (int a = 0; a < ld; a++) {
          double vk[3];
#pragma unroll
          for (int k = 0; k < 3; k++) vk[k] = k < ld ? V[(ot + a)*GG_LD + o + k] : 0.0;
#pragma unroll
          for (int c = 0; c < 6; c++) {
            double u = 0.0;
            for (int r = 0; r < rows; r++) u += f.J(r, f.lcol[t] + a)*f.J(r, f.pcol[s] + c);
#pragma unroll
            for (int k = 0; k < 3; k++) acc[c][k] += u*vk[k];
          }
        }
      }
#pragma unroll
      for (int c = 0; c < 6; c++)
#pragma unroll
        for (int k = 0; k < 3; k++) if (k < ld) atomicAdd(mq + (size_t)(c0 + c)*3 + k, acc[c][k]);
    }
    __threadfence_block();
    __syncwarp();
    for (int col = lane; col < j.nc; col += 32) {
      double zk[3] = {0.0, 0.0, 0.0};
      for (int r = 0; r < j.nc; r++) {
        const double x = j.xcc[(size_t)r*j.nc + col];
#pragma unroll
        for (int k = 0; k < 3; k++) zk[k] += __ldcg(mq + (size_t)r*3 + k)*x;
      }
      for (int k = 0; k < ld; k++) j.z[((size_t)q*3 + k)*j.nc + col] = -zk[k];
    }
  }
}
int launch_cov_strips(const StripJob& j, cudaStream_t s) {
  if (j.ng == 0) return 0;
  static bool attr = false;
  if (!attr) { cudaFuncSetAttribute(cov_strip_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)gg_smem()); attr = true; }
  cov_strip_kernel<<<general_grid(j.ng), 64, gg_smem(), s>>>(j);
  return 1;
}

int launch_cov_general(const GeneralGroups& G, const double* sig, int TPC, double* out_point, int* fail, cudaStream_t s) {
  if (G.n_groups == 0) return 0;
  static bool attr = false;
  if (!attr) { cudaFuncSetAttribute(cov_general_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)gg_smem()); attr = true; }
  cov_general_kernel<<<general_grid(G.n_groups), 64, gg_smem(), s>>>(G.blocks, G.gptr, (const FRef*)G.refs, G.gl0, G.gnl, G.n_groups, sig, TPC, out_point, fail);
  return 1;
}

int general_grid(int n_groups) { return (n_groups + 1)/2; }

int launch_schur_general(const GeneralGroups& G, const DevBand& B, double lambda, int* fail, cudaStream_t s) {
  if (G.n_groups == 0) return 0;
  static bool attr = false;
  if (!attr) { cudaFuncSetAttribute(schur_general_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)gg_smem());
               cudaFuncSetAttribute(backsub_general_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)gg_smem()); attr = true; }
  schur_general_kernel<<<general_grid(G.n_groups), 64, gg_smem(), s>>>(G.blocks, G.gptr, (const FRef*)G.refs, G.gl0, G.gnl, G.n_groups, B, lambda, fail);
  return 1;
}
int launch_backsub_general(const GeneralGroups& G, const DevBand& B, double lambda, double* dl_point, int nl_stride,
                           double* partials, cudaStream_t s) {
  if (G.n_groups == 0) return 0;
  static bool attr = false;
  if (!attr) { cudaFuncSetAttribute(schur_general_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)gg_smem());
               cudaFuncSetAttribute(backsub_general_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)gg_smem()); attr = true; }
  backsub_general_kernel<<<general_grid(G.n_groups), 64, gg_smem(), s>>>(G.blocks, G.gptr, (const FRef*)G.refs, G.gl0, G.gnl, G.n_groups, B, lambda, dl_point, nl_stride, partials);
  return 1;
}

}  // namespace dynoba
