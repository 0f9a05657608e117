// binaryop_math.cu — binop_kernel (binaryop.cuh) for TRUE_DIV, POW, INT_POW, LOG_BASE and ATAN2.
#include "binaryop.cuh"

namespace b2 {
namespace binop {

void launch_math(int op, int32_t ctype, const args& a, cudaStream_t stream)
{
  switch (op) {
    case B2_BINOP_TRUE_DIV: return launch_ctype<B2_BINOP_TRUE_DIV>(ctype, a, stream);
    case B2_BINOP_POW: return launch_ctype<B2_BINOP_POW>(ctype, a, stream);
    case B2_BINOP_INT_POW: return launch_ctype<B2_BINOP_INT_POW>(ctype, a, stream);
    case B2_BINOP_LOG_BASE: return launch_ctype<B2_BINOP_LOG_BASE>(ctype, a, stream);
    case B2_BINOP_ATAN2: return launch_ctype<B2_BINOP_ATAN2>(ctype, a, stream);
    default: B2_FAIL(B2_ERR_LOGIC, "binary_operation: operator outside the math family");
  }
}

}  // namespace binop
}  // namespace b2
