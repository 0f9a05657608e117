// binaryop_logical.cu — binop_kernel (binaryop.cuh) for LOGICAL_AND, LOGICAL_OR, NULL_LOGICAL_AND and NULL_LOGICAL_OR.
#include "binaryop.cuh"

namespace b2 {
namespace binop {

void launch_logical(int op, int32_t ctype, const args& a, cudaStream_t stream)
{
  switch (op) {
    case B2_BINOP_LOGICAL_AND: return launch_ctype<B2_BINOP_LOGICAL_AND>(ctype, a, stream);
    case B2_BINOP_LOGICAL_OR: return launch_ctype<B2_BINOP_LOGICAL_OR>(ctype, a, stream);
    case B2_BINOP_NULL_LOGICAL_AND: return launch_ctype<B2_BINOP_NULL_LOGICAL_AND>(ctype, a, stream);
    case B2_BINOP_NULL_LOGICAL_OR: return launch_ctype<B2_BINOP_NULL_LOGICAL_OR>(ctype, a, stream);
    default: B2_FAIL(B2_ERR_LOGIC, "binary_operation: operator outside the logical family");
  }
}

}  // namespace binop
}  // namespace b2
