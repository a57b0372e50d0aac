// stub: see tests/stubs/gtsam_stub.h.  gtsam/linear/JacobianFactor.h (4.2.0) with the block API the kept-landmark path of
// include/dynoba_gtsam_adapter.hpp reads: error(x) = 1/2 |A x - b|^2 (whitened by the model, when there is one);
// begin() / end() iterate over the keys (the Factor base), getA(it) is the block of the key at it, rows() the number of
// rows; the constructor takes a container of (key, block) pairs.  tests/test_window_landmarks.py puts this directory
// before tests/stubs on the include path.
#pragma once
#include <gtsam/linear/HessianFactor.h>

namespace gtsam {
using SharedDiagonal = boost::shared_ptr<noiseModel::Diagonal>;
class JacobianFactor : public GaussianFactor {
 public:
  using shared_ptr = boost::shared_ptr<JacobianFactor>;
  using const_iterator = KeyVector::const_iterator;
  template <typename TERMS> JacobianFactor(const TERMS& terms, const Vector& b, const SharedDiagonal& model = SharedDiagonal());
  const_iterator begin() const;
  const_iterator end() const;
  Matrix getA(const_iterator variable) const;
  Vector getb() const;
  const SharedDiagonal& get_model() const;
  std::size_t rows() const;
};
}  // namespace gtsam
