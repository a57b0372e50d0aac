// stub: see tests/stubs/gtsam_stub.h.  gtsam/linear/HessianFactor.h (4.2.0): error(x) = 1/2 x^T G x - x^T g + 1/2 f over
// the factor's keys in order, information() = G (dense, symmetric), linearTerm() = g, constantTerm() = f.  Also the
// GaussianFactor base and the Vector alias of gtsam/base/Vector.h (Eigen::VectorXd).
#pragma once
#include "../navigation/CombinedImuFactor.h"
#include "../inference/Key.h"

namespace gtsam {
struct Vector { long size() const; double operator()(long i) const; };   // Eigen::VectorXd
class GaussianFactor {
 public:
  using shared_ptr = boost::shared_ptr<GaussianFactor>;
  virtual ~GaussianFactor();
  const KeyVector& keys() const;
};
class JacobianFactor;
class HessianFactor : public GaussianFactor {
 public:
  using shared_ptr = boost::shared_ptr<HessianFactor>;
  // Gs: the upper-triangular blocks G_11, G_12, ..., G_1n, G_22, ... in row order; gs: one block of g per key
  HessianFactor(const KeyVector& js, const std::vector<Matrix>& Gs, const std::vector<Vector>& gs, double f);
  explicit HessianFactor(const JacobianFactor& cg);
  Matrix information() const;
  Vector linearTerm() const;
  double constantTerm() const;
};
}  // namespace gtsam
