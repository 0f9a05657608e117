// binaryop_arith.cu — binop_kernel (binaryop.cuh) for ADD, SUB, MUL, DIV, FLOOR_DIV, MOD, PMOD, PYMOD, NULL_MAX and NULL_MIN.
#include "binaryop.cuh"

namespace b2 {
namespace binop {

void launch_arith(int op, int32_t ctype, const args& a, cudaStream_t stream)
{
  switch (op) {
    case B2_BINOP_ADD: return launch_ctype<B2_BINOP_ADD>(ctype, a, stream);
    case B2_BINOP_SUB: return launch_ctype<B2_BINOP_SUB>(ctype, a, stream);
    case B2_BINOP_MUL: return launch_ctype<B2_BINOP_MUL>(ctype, a, stream);
    case B2_BINOP_DIV: return launch_ctype<B2_BINOP_DIV>(ctype, a, stream);
    case B2_BINOP_FLOOR_DIV: return launch_ctype<B2_BINOP_FLOOR_DIV>(ctype, a, stream);
    case B2_BINOP_MOD: return launch_ctype<B2_BINOP_MOD>(ctype, a, stream);
    case B2_BINOP_PMOD: return launch_ctype<B2_BINOP_PMOD>(ctype, a, stream);
    case B2_BINOP_PYMOD: return launch_ctype<B2_BINOP_PYMOD>(ctype, a, stream);
    case B2_BINOP_NULL_MAX: return launch_ctype<B2_BINOP_NULL_MAX>(ctype, a, stream);
    case B2_BINOP_NULL_MIN: return launch_ctype<B2_BINOP_NULL_MIN>(ctype, a, stream);
    default: B2_FAIL(B2_ERR_LOGIC, "binary_operation: operator outside the arith family");
  }
}

}  // namespace binop
}  // namespace b2
