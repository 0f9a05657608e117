// cudf/replace.hpp — see cudf/detail/b2_bridge.hpp (header-only wrappers over include/cudf_b200.h)
#pragma once
#include "detail/b2_bridge.hpp"
