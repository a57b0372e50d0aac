// stub: see tests/stubs/gtsam_stub.h.  gtsam/linear/GaussianFactorGraph.h (4.2.0): FactorGraph<GaussianFactor>
#pragma once
#include "HessianFactor.h"

namespace gtsam {
class GaussianFactorGraph { public: void push_back(const GaussianFactor::shared_ptr& factor); std::size_t size() const; };
}  // namespace gtsam
