// triangulate_host.cu -- the triangulation of dynosam_b200/csrc/triangulate.cuh compiled for the host, so that
// tests/test_triangulate.py can run it on a machine without a GPU and tools/triangulate_bench.py can time it on one CPU
// thread.  The problem loop is the builder's CPU path: tri_solve over the emulated lanes of TriHostLanes.
#include <vector>
#include "triangulate.cuh"

using namespace dynoba;

extern "C" {
// every problem of a batch, the arguments of dynoba_triangulate_batch (no validation: the tests pass valid input)
void host_triangulate_batch(int n, const int* off, const double* poses, const double* kp, const double* calib5, double rank_tol,
                            double thr, double* point, int* status, double* reproj, double* sv) {
  std::vector<double> A;
  for (int p = 0; p < n; p++) {
    const int m = off[p + 1] - off[p];
    A.resize(8*(size_t)(m > 0 ? m : 1));
    TriHostLanes lanes; TriOut o;
    tri_solve(m, poses + 12*(size_t)off[p], kp + 2*(size_t)off[p], calib5 + 5*(size_t)p, rank_tol, thr, A.data(), lanes, o);
    status[p] = o.status; reproj[p] = o.reproj;
    for (int k = 0; k < 3; k++) point[3*p + k] = o.point[k];
    for (int k = 0; k < 4; k++) sv[4*p + k] = o.sv[k];
  }
}
}
