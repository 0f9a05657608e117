// binaryop_bits.cu — binop_kernel (binaryop.cuh) for the shifts and the bitwise operators.
#include "binaryop.cuh"

namespace b2 {
namespace binop {

void launch_bits(int op, int32_t ctype, const args& a, cudaStream_t stream)
{
  switch (op) {
    case B2_BINOP_SHIFT_LEFT: return launch_ctype<B2_BINOP_SHIFT_LEFT>(ctype, a, stream);
    case B2_BINOP_SHIFT_RIGHT: return launch_ctype<B2_BINOP_SHIFT_RIGHT>(ctype, a, stream);
    case B2_BINOP_SHIFT_RIGHT_UNSIGNED: return launch_ctype<B2_BINOP_SHIFT_RIGHT_UNSIGNED>(ctype, a, stream);
    case B2_BINOP_BITWISE_AND: return launch_ctype<B2_BINOP_BITWISE_AND>(ctype, a, stream);
    case B2_BINOP_BITWISE_OR: return launch_ctype<B2_BINOP_BITWISE_OR>(ctype, a, stream);
    case B2_BINOP_BITWISE_XOR: return launch_ctype<B2_BINOP_BITWISE_XOR>(ctype, a, stream);
    default: B2_FAIL(B2_ERR_LOGIC, "binary_operation: operator outside the bits family");
  }
}

}  // namespace binop
}  // namespace b2
