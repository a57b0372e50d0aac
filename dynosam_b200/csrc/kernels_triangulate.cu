// kernels_triangulate.cu -- dynoba_triangulate_batch: the triangulation of triangulate.cuh for every problem of a batch in
// one launch, one warp per problem.
//
// A's rows are strided over the lanes (row r on lane r mod 32) and stored in the workspace, so the number of cameras is not
// limited; each lane writes and reads only its own rows.  V (4x4) is replicated in every lane's registers.  The column
// dots and norms of each rotation meet in a fixed butterfly of __shfl_xor_sync, which leaves the same bits in every lane:
// the warp's control flow stays uniform, and a problem's result depends on nothing but its own inputs.  This file is
// compiled with -fmad=false so that its arithmetic is the host build's operation for operation.
#include "internal.cuh"
#include "triangulate.cuh"

namespace dynoba {

constexpr int TRI_WARPS = 4;                    // problems per CTA

struct TriBatch {
  const int* off; const double* poses; const double* kp; const double* calib; double* A;
  double* point; int* status; double* reproj; double* sv;
  int n; double rank_tol, thr;
};

struct TriWarpLanes {
  int lane;
  template <class F> __device__ void each(F f) { f(lane); }
  template <int N, class F> __device__ void sum(F f, double* out) {
    double part[N];
    f(lane, part);
    for (int k = 0; k < N; k++) {
      double x = part[k];
      for (int o = TRI_LANES/2; o > 0; o >>= 1) x = x + __shfl_xor_sync(0xffffffffu, x, o);
      out[k] = x;
    }
  }
};

__global__ void __launch_bounds__(TRI_WARPS*32) triangulate_kernel(TriBatch B) {
  const int p = blockIdx.x*TRI_WARPS + (threadIdx.x >> 5);
  if (p >= B.n) return;                         // whole warps only: the kernel has no CTA-wide barrier
  TriWarpLanes lanes{ (int)(threadIdx.x & 31) };
  const int c0 = B.off[p], m = B.off[p + 1] - c0;
  TriOut o;
  tri_solve(m, B.poses + 12*(size_t)c0, B.kp + 2*(size_t)c0, B.calib + 5*(size_t)p, B.rank_tol, B.thr, B.A + 8*(size_t)c0,
            lanes, o);
  if (lanes.lane == 0) {
    B.status[p] = o.status; B.reproj[p] = o.reproj;
    for (int k = 0; k < 3; k++) B.point[3*(size_t)p + k] = o.point[k];
    for (int k = 0; k < 4; k++) B.sv[4*(size_t)p + k] = o.sv[k];
  }
}

static bool finite_all(const double* a, size_t n) {
  for (size_t i = 0; i < n; i++) if (!std::isfinite(a[i])) return false;
  return true;
}

}  // namespace dynoba

using namespace dynoba;

extern "C" {

int dynoba_triangulate_batch(int device, int32_t n_problems, const int32_t* offsets, const double* poses, const double* kp,
                             const double* calib5, double rank_tol, double reproj_threshold, double* point_out,
                             int32_t* status, double* reproj_norm, double* sv_out) {
  if (n_problems == 0) return DYNOBA_OK;
  if (n_problems < 0 || n_problems >= (1 << 24) || !offsets || !poses || !kp || !calib5 || !status) return DYNOBA_ERR_BAD_ARG;
  if (!std::isfinite(rank_tol) || rank_tol < 0.0 || std::isnan(reproj_threshold) || reproj_threshold < 0.0) return DYNOBA_ERR_BAD_ARG;
  if (offsets[0] != 0) return DYNOBA_ERR_BAD_ARG;
  for (int p = 0; p < n_problems; p++) if (offsets[p + 1] < offsets[p]) return DYNOBA_ERR_BAD_ARG;
  if (offsets[n_problems] > (1 << 27)) return DYNOBA_ERR_BAD_ARG;
  const size_t np = (size_t)n_problems, nc = (size_t)offsets[n_problems];
  if (!finite_all(poses, 12*nc) || !finite_all(kp, 2*nc) || !finite_all(calib5, 5*np)) return DYNOBA_ERR_BAD_ARG;
  for (size_t p = 0; p < np; p++) if (!(calib5[5*p] > 0.0) || !(calib5[5*p + 1] > 0.0)) return DYNOBA_ERR_BAD_ARG;
  if (device < 0 || device >= 64) return DYNOBA_ERR_CUDA;
  StarContext& ctx = star_context(device);
  std::lock_guard<std::mutex> lock(ctx.mu);
  int rc = star_device_ready(device); if (rc) return rc;
  DeviceBlock blk; TriBatch S{};
  int* d_off; double *d_pose, *d_kp, *d_cal;
  auto layout = [&]() {
    d_off = blk.take<int>(np + 1); d_pose = blk.take<double>(12*nc); d_kp = blk.take<double>(2*nc); d_cal = blk.take<double>(5*np);
    S.A = blk.take<double>(8*nc);
    S.point = blk.take<double>(3*np); S.status = blk.take<int>(np); S.reproj = blk.take<double>(np); S.sv = blk.take<double>(4*np);
  };
  layout();
  if (!blk.allocate(ctx)) { cudaGetLastError(); return DYNOBA_ERR_CUDA; }
  layout();
  cudaStream_t s = ctx.stream;
  cudaMemcpyAsync(d_off, offsets, 4*(np + 1), cudaMemcpyHostToDevice, s);
  if (nc) {
    cudaMemcpyAsync(d_pose, poses, 96*nc, cudaMemcpyHostToDevice, s);
    cudaMemcpyAsync(d_kp, kp, 16*nc, cudaMemcpyHostToDevice, s);
  }
  cudaMemcpyAsync(d_cal, calib5, 40*np, cudaMemcpyHostToDevice, s);
  S.off = d_off; S.poses = d_pose; S.kp = d_kp; S.calib = d_cal; S.n = n_problems; S.rank_tol = rank_tol; S.thr = reproj_threshold;
  triangulate_kernel<<<(n_problems + TRI_WARPS - 1)/TRI_WARPS, TRI_WARPS*32, 0, s>>>(S);
  cudaMemcpyAsync(status, S.status, 4*np, cudaMemcpyDeviceToHost, s);
  if (point_out) cudaMemcpyAsync(point_out, S.point, 24*np, cudaMemcpyDeviceToHost, s);
  if (reproj_norm) cudaMemcpyAsync(reproj_norm, S.reproj, 8*np, cudaMemcpyDeviceToHost, s);
  if (sv_out) cudaMemcpyAsync(sv_out, S.sv, 32*np, cudaMemcpyDeviceToHost, s);
  const cudaError_t e1 = cudaStreamSynchronize(s), e2 = cudaGetLastError();
  return (e1 == cudaSuccess && e2 == cudaSuccess) ? DYNOBA_OK : DYNOBA_ERR_CUDA;
}

}  // extern "C"
