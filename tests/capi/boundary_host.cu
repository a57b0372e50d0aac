// boundary_host.cu -- the object boundary mask of dynosam_b200/frontend_csrc/boundary.cuh compiled for the host, so that
// tests/test_object_boundary.py can run it on a machine without a GPU.  host_boundary runs boundary_seq, the sequential
// statement the kernels of frontend.cu parallelise, and boundary_finish, the host half of dynofront_object_boundary.
#include <vector>
#include "boundary.cuh"

extern "C" {
// the element's row half widths for radius r: hw[0..r]
void host_boundary_ellipse(int r, int* hw) { for (int dy = 0; dy <= r; dy++) hw[dy] = boundary_ellipse_hw(r, dy); }
int host_boundary_thickness(int W, int H) { return boundary_thickness(W, H); }
// the whole call (labels are not checked: the tests pass labels in [0, 255]); returns the number of objects
int host_boundary(const int32_t* M, int W, int H, int t, int capacity, int32_t* objects, int32_t* bb, int32_t* inner_bb, uint8_t* boundary) {
  std::vector<uint8_t> T((size_t)W*H);
  std::vector<int> bb_ext(4*(BOUNDARY_MAX_LABEL + 1), 0), inner_ext(4*(BOUNDARY_MAX_LABEL + 1), 0);
  boundary_seq(M, W, H, t, T.data(), boundary, bb_ext.data(), inner_ext.data());
  return boundary_finish(bb_ext.data(), inner_ext.data(), W, H, capacity, objects, bb, inner_bb);
}
}
