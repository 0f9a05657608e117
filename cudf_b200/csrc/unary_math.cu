// unary_math.cu — unary_kernel (unary.cuh) for SIN .. ABS and RINT: FLOAT32 / FLOAT64 on the vector path, the integer types
// and BOOL8 computed in double (ABS: in int64 / uint64) on the generic path.
#include "unary.cuh"

namespace b2 {
namespace unary {
namespace {

template <int OP>
void launch_op(const args& a, cudaStream_t stream)
{
  if (a.in_type == B2_FLOAT32) return launch<math_fn<OP>, float, float, float>(a, stream);
  if (a.in_type == B2_FLOAT64) return launch<math_fn<OP>, double, double, double>(a, stream);
  if constexpr (OP == B2_UNARY_ABS) {
    if (is_signed_id(a.in_type)) return launch<math_fn<OP>, int64_t, rt, rt>(a, stream);
    return launch<math_fn<OP>, uint64_t, rt, rt>(a, stream);
  } else if constexpr (OP != B2_UNARY_RINT) {
    return launch<math_fn<OP>, double, rt, rt>(a, stream);
  }
  B2_FAIL(B2_ERR_LOGIC, "unary_operation: no math kernel for this type");
}

}  // namespace

void launch_math(int op, const args& a, cudaStream_t stream)
{
  switch (op) {
    case B2_UNARY_SIN: return launch_op<B2_UNARY_SIN>(a, stream);
    case B2_UNARY_COS: return launch_op<B2_UNARY_COS>(a, stream);
    case B2_UNARY_TAN: return launch_op<B2_UNARY_TAN>(a, stream);
    case B2_UNARY_ARCSIN: return launch_op<B2_UNARY_ARCSIN>(a, stream);
    case B2_UNARY_ARCCOS: return launch_op<B2_UNARY_ARCCOS>(a, stream);
    case B2_UNARY_ARCTAN: return launch_op<B2_UNARY_ARCTAN>(a, stream);
    case B2_UNARY_SINH: return launch_op<B2_UNARY_SINH>(a, stream);
    case B2_UNARY_COSH: return launch_op<B2_UNARY_COSH>(a, stream);
    case B2_UNARY_TANH: return launch_op<B2_UNARY_TANH>(a, stream);
    case B2_UNARY_ARCSINH: return launch_op<B2_UNARY_ARCSINH>(a, stream);
    case B2_UNARY_ARCCOSH: return launch_op<B2_UNARY_ARCCOSH>(a, stream);
    case B2_UNARY_ARCTANH: return launch_op<B2_UNARY_ARCTANH>(a, stream);
    case B2_UNARY_EXP: return launch_op<B2_UNARY_EXP>(a, stream);
    case B2_UNARY_LOG: return launch_op<B2_UNARY_LOG>(a, stream);
    case B2_UNARY_SQRT: return launch_op<B2_UNARY_SQRT>(a, stream);
    case B2_UNARY_CBRT: return launch_op<B2_UNARY_CBRT>(a, stream);
    case B2_UNARY_CEIL: return launch_op<B2_UNARY_CEIL>(a, stream);
    case B2_UNARY_FLOOR: return launch_op<B2_UNARY_FLOOR>(a, stream);
    case B2_UNARY_ABS: return launch_op<B2_UNARY_ABS>(a, stream);
    case B2_UNARY_RINT: return launch_op<B2_UNARY_RINT>(a, stream);
    default: B2_FAIL(B2_ERR_LOGIC, "unary_operation: operator outside the math family");
  }
}

}  // namespace unary
}  // namespace b2
