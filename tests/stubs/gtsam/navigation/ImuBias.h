// stub: see tests/stubs/gtsam_stub.h.  gtsam/navigation/ImuBias.h (4.2.0) and the Vector3 alias of geometry/Point3.h:
// in GTSAM 4.2 Point3 IS Eigen::Vector3d, so a velocity value and a landmark value have the same C++ type.
#pragma once
#include "../../gtsam_stub.h"

namespace gtsam {
using Vector3 = Point3;
namespace imuBias {
class ConstantBias {
 public:
  ConstantBias(); ConstantBias(const Vector3& acc, const Vector3& gyro);
  const Vector3& accelerometer() const; const Vector3& gyroscope() const;
};
}  // namespace imuBias
}  // namespace gtsam
