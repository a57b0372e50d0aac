#pragma once
#include "../../gtsam_stub.h"
namespace gtsam { using KeyVector = std::vector<Key>; }
