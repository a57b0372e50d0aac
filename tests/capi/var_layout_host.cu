// var_layout_host.cu -- the variable layout of dynosam_b200/csrc/var_layout.cuh compiled for the host, so that
// tests/test_var_layout.py can run it on a machine without a GPU.
#include "var_layout.cuh"

using namespace dynoba;

static VarLayout L;         // the layout of the latest host_set_layout call

extern "C" {
// n = [np, npt, nfl, nv, nb]; pos, pt_new, fl_new as finalize leaves them; out = the stride of every kind's SoA image
void host_set_layout(const int64_t* n, const int32_t* pos, const int32_t* pt_new, const int32_t* fl_new, int32_t* out) {
  L = VarLayout{n[0], n[1], n[2], n[3], n[4]};
  L.pos.assign(pos, pos + L.NP()); L.pt_new.assign(pt_new, pt_new + L.npt); L.fl_new.assign(fl_new, fl_new + L.nfl);
  for (int k = 0; k < NUM_KINDS; k++) out[k] = L.stride(k);
}
// [width, tdim, rows, poselike] of every kind
void host_kinds(int32_t* out) { for (int k = 0; k < NUM_KINDS; k++) { const KindInfo K = KINDS[k]; out[4*k] = K.width; out[4*k + 1] = K.tdim; out[4*k + 2] = K.rows; out[4*k + 3] = K.poselike; } }
// pos of the counts set last and the hints of the poses, velocities and biases (nullptr: none)
void host_poselike_positions(const int32_t* hint, const int32_t* vhint, const int32_t* bhint, int32_t* pos) {
  std::vector<int32_t> hints[NUM_KINDS];
  const int32_t* h[NUM_KINDS] = {hint, nullptr, nullptr, vhint, bhint};
  for (int k = 0; k < NUM_KINDS; k++) if (h[k]) hints[k].assign(h[k], h[k] + L.count(k));
  const std::vector<int32_t> p = L.poselike_positions(hints);
  std::copy(p.begin(), p.end(), pos);
}
int32_t host_column_checked(int kind, int64_t i) { return L.column_checked(kind, i); }
void host_blank_image(int kind, double* img) { const std::vector<double> b = L.blank_image(kind); std::copy(b.begin(), b.end(), img); }
void host_scatter_values(int kind, const double* vals, double* img) { L.scatter_values(kind, vals, img); }
void host_gather_values(int kind, const double* img, double* vals) { L.gather_values(kind, img, vals); }
// the two directions of dynoba_retract and dynoba_solve
void host_scatter_delta(const double* delta, double* r, double* pt, double* fl) { L.walk_delta(r, pt, fl, [&](size_t u, double& v) { v = delta[u]; }); }
void host_gather_delta(double* r, double* pt, double* fl, double* delta) { L.walk_delta(r, pt, fl, [&](size_t u, double& v) { delta[u] = v; }); }
int64_t host_reduced_map(int32_t* m) { const std::vector<int32_t> v = L.reduced_map(); std::copy(v.begin(), v.end(), m); return L.reduced_dim(); }
// slot [n][4] and sidx [sum of tangent dimensions]
void host_prior_table(int n, const int32_t* kind, const int32_t* idx, int32_t* slot, int32_t* sidx) {
  std::vector<int4> s; std::vector<int32_t> x;
  L.prior_table(n, kind, idx, s, x);
  for (int i = 0; i < n; i++) { slot[4*i] = s[i].x; slot[4*i + 1] = s[i].y; slot[4*i + 2] = s[i].z; slot[4*i + 3] = s[i].w; }
  std::copy(x.begin(), x.end(), sidx);
}
// [nv + nb][2]
void host_nav_table(int32_t* nav) {
  const std::vector<int2> v = L.nav_table();
  for (size_t i = 0; i < v.size(); i++) { nav[2*i] = v[i].x; nav[2*i + 1] = v[i].y; }
}
}
