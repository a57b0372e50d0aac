// stub: see tests/stubs/gtsam_stub.h.  gtsam/navigation/CombinedImuFactor.h (4.2.0, GTSAM_TANGENT_PREINTEGRATION=OFF:
// PreintegratedCombinedMeasurements derives from ManifoldPreintegration), noiseModel::Gaussian::R().
#pragma once
#include "ImuBias.h"

namespace gtsam {
struct Matrix { long rows() const; long cols() const; double operator()(long r, long c) const; };   // Eigen::MatrixXd
namespace noiseModel {
class Gaussian : public Base { public: Matrix R() const; };
}  // namespace noiseModel
// boost::optional<Vector3> of PreintegrationParams::omegaCoriolis
struct OptionalVector3 { explicit operator bool() const; const Vector3& operator*() const; };
struct PreintegrationCombinedParams { Vector3 n_gravity; OptionalVector3 omegaCoriolis; bool use2ndOrderCoriolis; };
class PreintegratedCombinedMeasurements {
 public:
  Rot3 deltaRij() const; Vector3 deltaPij() const; Vector3 deltaVij() const; double deltaTij() const;
  const imuBias::ConstantBias& biasHat() const;
  const Matrix3& delRdelBiasOmega() const; const Matrix3& delPdelBiasAcc() const; const Matrix3& delPdelBiasOmega() const;
  const Matrix3& delVdelBiasAcc() const; const Matrix3& delVdelBiasOmega() const;
  const PreintegrationCombinedParams& p() const;
};
class CombinedImuFactor : public NoiseModelFactor {
 public:
  Key key1() const; Key key2() const; Key key3() const; Key key4() const; Key key5() const; Key key6() const;
  const PreintegratedCombinedMeasurements& preintegratedMeasurements() const;
};
}  // namespace gtsam
