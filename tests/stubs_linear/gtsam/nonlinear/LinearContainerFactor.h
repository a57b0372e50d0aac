// stub: see tests/stubs/gtsam_stub.h.  gtsam/nonlinear/LinearContainerFactor.h (4.2.0): a GaussianFactor wrapped as a
// NonlinearFactor, with the Values it was linearised at (boost::optional<Values> in GTSAM; the constructors keep only the
// factor's keys of the Values they are given)
// (tests/stubs/gtsam/nonlinear/LinearContainerFactor.h with include paths, so that it takes the JacobianFactor of this
// directory)
#pragma once
#include <gtsam/linear/GaussianFactorGraph.h>
#include <gtsam/linear/HessianFactor.h>
#include <gtsam/linear/JacobianFactor.h>
#include <gtsam/nonlinear/NonlinearFactorGraph.h>
#include <gtsam/nonlinear/Values.h>

namespace gtsam {
struct OptionalValues { explicit operator bool() const; const Values& operator*() const; const Values* operator->() const; };
class LinearContainerFactor : public NonlinearFactor {
 public:
  LinearContainerFactor(const HessianFactor& factor, const Values& linearizationPoint);
  static NonlinearFactorGraph ConvertLinearGraph(const GaussianFactorGraph& linear_graph, const Values& linearizationPoint);
  const GaussianFactor::shared_ptr& factor() const;
  const OptionalValues& linearizationPoint() const;
  bool hasLinearizationPoint() const;
};
}  // namespace gtsam
