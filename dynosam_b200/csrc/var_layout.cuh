// var_layout.cuh -- where every variable sits: the one map between the caller's order of each variable kind and the
// solver's layout (pose-like positions, landmark device indices, the SoA images of DevVars, the band scalars), and the
// caller layouts include/dynoba.h documents.  Plain host code, so that tests/capi/var_layout_host.cu can run it on a
// machine without a GPU.
#pragma once
#include <parallel/algorithm>
#include <omp.h>
#include <algorithm>
#include <cstdint>
#include <numeric>
#include <tuple>
#include <vector>
#include "internal.cuh"

namespace dynoba {

static_assert(VC_POSE == (int)DYNOBA_POSE6 && VC_POINT == (int)DYNOBA_POINT3 && VC_FLOW == (int)DYNOBA_FLOW2 &&
              VC_VEL == (int)DYNOBA_VEL3 && VC_BIAS == (int)DYNOBA_BIAS6, "factor slot classes and variable kinds share one numbering");

// Per kind: doubles of a value in the caller's arrays, tangent dimension, rows of its SoA image (velocities and biases sit
// in the 12-row pose image), and whether it is pose-like (a 6-wide band block; a velocity's last 3 scalars are inert).
struct KindInfo { int width, tdim, rows; bool poselike; };
constexpr int NUM_KINDS = 5;
inline constexpr KindInfo KINDS[NUM_KINDS] = { {12, 6, 12, true}, {3, 3, 3, false}, {2, 2, 2, false}, {3, 3, 12, true}, {6, 6, 12, true} };
constexpr bool kinds_agree(int k = 0) { return k == NUM_KINDS || (KINDS[k].tdim == class_dim(k) && KINDS[k].poselike == is_poselike(k) && kinds_agree(k + 1)); }
static_assert(kinds_agree(), "KINDS and factors.cuh disagree");
inline bool valid_kind(int kind) { return kind >= 0 && kind < NUM_KINDS; }
inline bool poselike_kind(int kind) { return valid_kind(kind) && KINDS[kind].poselike; }
inline int pad32(int64_t n) { return (int)((n + 31)/32*32); }

// pos[j] = position of item j in the stable order of n items by `less`
template <class Less> std::vector<int32_t> positions_by(int64_t n, Less less) {
  std::vector<int32_t> ord(n), pos(n);
  std::iota(ord.begin(), ord.end(), 0);
  int unsorted = 0;
#pragma omp parallel for schedule(static) reduction(|:unsorted)
  for (int64_t i = 1; i < n; i++) unsorted |= less((int32_t)i, (int32_t)(i - 1));
  if (unsorted) __gnu_parallel::stable_sort(ord.begin(), ord.end(), less);
#pragma omp parallel for schedule(static)
  for (int64_t i = 0; i < n; i++) pos[ord[i]] = (int32_t)i;
  return pos;
}

// pos: solver position of every pose-like variable, indexed [poses | velocities | biases]; pt_new / fl_new: device index
// of every point / flow.
struct VarLayout {
  int64_t np = 0, npt = 0, nfl = 0, nv = 0, nb = 0;
  std::vector<int32_t> pos, pt_new, fl_new;

  int64_t NP() const { return np + nv + nb; }
  int64_t first(int kind) const { return kind == DYNOBA_BIAS6 ? np + nv : (kind == DYNOBA_VEL3 ? np : 0); }   // of a pose-like kind in pos
  int64_t count(int kind) const { const int64_t n[NUM_KINDS] = {np, npt, nfl, nv, nb}; return n[kind]; }
  int stride(int kind) const { return pad32(KINDS[kind].poselike ? NP() : count(kind)); }     // of the kind's SoA image
  size_t image_size(int kind) const { return (size_t)KINDS[kind].rows*stride(kind); }
  // SoA column of variable i of a kind: its solver position (pose-like) or device index (landmarks)
  int32_t column(int kind, int64_t i) const { return kind == DYNOBA_POINT3 ? pt_new[i] : (kind == DYNOBA_FLOW2 ? fl_new[i] : pos[first(kind) + i]); }
  // the same for a kind and an index from outside the library: -1 when out of range
  int32_t column_checked(int kind, int64_t i) const { return valid_kind(kind) && i >= 0 && i < count(kind) ? column(kind, i) : -1; }

  // pos for the order hints of the pose-like kinds (hints[kind] = rank of every variable of the kind, or empty): ordered
  // by (rank, kind: pose < velocity < bias, index).  A kind without a hint ranks by index, so X_k, V_k, b_k with the frame
  // as rank sit next to each other and the reduced system stays banded.
  std::vector<int32_t> poselike_positions(const std::vector<int32_t>* hints) const {
    std::vector<std::tuple<int32_t, int, int32_t>> key(NP());
    for (int kind : {DYNOBA_POSE6, DYNOBA_VEL3, DYNOBA_BIAS6})
      for (int32_t i = 0; i < count(kind); i++) key[first(kind) + i] = std::make_tuple(hints[kind].empty() ? i : hints[kind][i], kind, i);
    return positions_by(NP(), [&](int32_t a, int32_t b) { return key[a] < key[b]; });
  }

  // Values: caller array [count][width] <-> SoA image [rows][stride].  A fresh image is zero, with the identity in
  // every column of the pose image; a scatter writes every row of its columns (0 past the width).
  std::vector<double> blank_image(int kind) const {
    std::vector<double> img(image_size(kind), 0.0);
    const int st = stride(kind);
    if (KINDS[kind].rows == 12) for (int p = 0; p < st; p++) img[p] = img[(size_t)4*st + p] = img[(size_t)8*st + p] = 1.0;
    return img;
  }
  void scatter_values(int kind, const double* vals, double* img) const {
    const KindInfo K = KINDS[kind]; const int st = stride(kind);
    for (int64_t i = 0; i < count(kind); i++) {
      const int32_t p = column(kind, i);
      for (int k = 0; k < K.rows; k++) img[(size_t)k*st + p] = k < K.width ? vals[i*K.width + k] : 0.0;
    }
  }
  void gather_values(int kind, const double* img, double* vals) const {
    const KindInfo K = KINDS[kind]; const int st = stride(kind);
    for (int64_t i = 0; i < count(kind); i++) {
      const int32_t p = column(kind, i);
      for (int k = 0; k < K.width; k++) vals[i*K.width + k] = img[(size_t)k*st + p];
    }
  }

  // f(kind, i, c) for tangent scalar c of every variable i of the listed kinds, in the order of the list
  template <class F> void walk(std::initializer_list<int> kinds, F f) const {
    for (int kind : kinds) for (int64_t i = 0; i < count(kind); i++) for (int c = 0; c < KINDS[kind].tdim; c++) f(kind, i, c);
  }
  // f(u, s) for every scalar of the delta of dynoba_solve / dynoba_retract: u = its index in [poses 6 | points 3 | flows 2
  // | velocities 3 | biases 6] (caller order), s = the same scalar in the band vector r or the point / flow delta images
  template <class F> void walk_delta(double* r, double* pt, double* fl, F f) const {
    size_t u = 0;
    walk({DYNOBA_POSE6, DYNOBA_POINT3, DYNOBA_FLOW2, DYNOBA_VEL3, DYNOBA_BIAS6}, [&](int kind, int64_t i, int c) {
      const size_t p = column(kind, i);
      f(u++, kind == DYNOBA_POINT3 ? pt[(size_t)c*stride(kind) + p] : (kind == DYNOBA_FLOW2 ? fl[(size_t)c*stride(kind) + p] : r[6*p + c]));
    });
  }
  // the reduced system in the caller layout [poses 6 | velocities 3 | biases 6]: its dimension, and the map band scalar
  // -> index there (-1 for the inert scalars of a velocity)
  int64_t reduced_dim() const { return 6*np + 3*nv + 6*nb; }
  std::vector<int32_t> reduced_map() const {
    std::vector<int32_t> m((size_t)6*NP(), -1);
    int32_t u = 0;
    walk({DYNOBA_POSE6, DYNOBA_VEL3, DYNOBA_BIAS6}, [&](int kind, int64_t i, int c) { m[6*(size_t)column(kind, i) + c] = u++; });
    return m;
  }

  // A prior over n pose-like variables (indices checked by the caller): slot i = (kind, position, offset of its value in
  // the prior's lin, offset of its scalars in sidx); sidx = the band scalar of every tangent scalar, in slot order.
  void prior_table(int n, const int32_t* kind, const int32_t* idx, std::vector<int4>& slot, std::vector<int32_t>& sidx) const {
    for (int i = 0, lo = 0; i < n; lo += KINDS[kind[i]].width, i++) {
      const int32_t p = column(kind[i], idx[i]);
      slot.push_back(make_int4(kind[i], p, lo, (int)sidx.size()));
      for (int c = 0; c < KINDS[kind[i]].tdim; c++) sidx.push_back(6*p + c);
    }
  }
  // (position, tangent dimension) of every velocity, then every bias
  std::vector<int2> nav_table() const {
    std::vector<int2> nav;
    for (int kind : {DYNOBA_VEL3, DYNOBA_BIAS6}) for (int64_t i = 0; i < count(kind); i++) nav.push_back(make_int2(column(kind, i), KINDS[kind].tdim));
    return nav;
  }
};

// the device SoA image that holds a kind
inline double* image_of(const DevVars& V, int kind) { return KINDS[kind].poselike ? V.pose : (kind == DYNOBA_POINT3 ? V.point : V.flow); }

}  // namespace dynoba
