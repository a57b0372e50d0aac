// stub: see tests/stubs/gtsam_stub.h.  gtsam/linear/JacobianFactor.h (4.2.0)
#pragma once
#include "HessianFactor.h"

namespace gtsam {
class JacobianFactor : public GaussianFactor { public: using shared_ptr = boost::shared_ptr<JacobianFactor>; };
}  // namespace gtsam
