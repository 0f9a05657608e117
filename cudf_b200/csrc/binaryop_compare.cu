// binaryop_compare.cu — binop_kernel (binaryop.cuh) for the six comparisons, NULL_EQUALS and NULL_NOT_EQUALS.
#include "binaryop.cuh"

namespace b2 {
namespace binop {

void launch_compare(int op, int32_t ctype, const args& a, cudaStream_t stream)
{
  switch (op) {
    case B2_BINOP_EQUAL: return launch_ctype<B2_BINOP_EQUAL>(ctype, a, stream);
    case B2_BINOP_NOT_EQUAL: return launch_ctype<B2_BINOP_NOT_EQUAL>(ctype, a, stream);
    case B2_BINOP_LESS: return launch_ctype<B2_BINOP_LESS>(ctype, a, stream);
    case B2_BINOP_GREATER: return launch_ctype<B2_BINOP_GREATER>(ctype, a, stream);
    case B2_BINOP_LESS_EQUAL: return launch_ctype<B2_BINOP_LESS_EQUAL>(ctype, a, stream);
    case B2_BINOP_GREATER_EQUAL: return launch_ctype<B2_BINOP_GREATER_EQUAL>(ctype, a, stream);
    case B2_BINOP_NULL_EQUALS: return launch_ctype<B2_BINOP_NULL_EQUALS>(ctype, a, stream);
    case B2_BINOP_NULL_NOT_EQUALS: return launch_ctype<B2_BINOP_NULL_NOT_EQUALS>(ctype, a, stream);
    default: B2_FAIL(B2_ERR_LOGIC, "binary_operation: operator outside the compare family");
  }
}

}  // namespace binop
}  // namespace b2
