// binaryop.cu — cudf::binary_operation over fixed-width columns and scalars (cpp/include/cudf/binaryop.hpp,
// cpp/src/binaryop/binaryop.cpp and cpp/src/binaryop/compiled/ of the reference): the type rules, the checks, the output
// column and one launch of binop_kernel (binaryop.cuh) for the operator's family.
//
// Unlike the reference (bitmask_and, then the operator, then a null_count pass) one kernel writes values, mask and null
// count. The only read-back is a scalar operand's validity, which decides whether the output needs a mask at all.
#include "binaryop.cuh"

namespace b2 {
namespace {

using namespace binop;

constexpr int32_t NUM_TYPE_IDS = 29;  // cudf::type_id::NUM_TYPE_IDS

bool is_chrono(int32_t id) { return id >= B2_TIMESTAMP_DAYS && id <= B2_DURATION_NANOSECONDS; }

// std::common_type of two of INT8..BOOL8: the usual arithmetic conversions after integral promotion, except that a type
// paired with itself stays itself
int32_t common_type(int32_t a, int32_t b)
{
  if (a == b) return a;
  if (a == B2_FLOAT64 || b == B2_FLOAT64) return B2_FLOAT64;
  if (a == B2_FLOAT32 || b == B2_FLOAT32) return B2_FLOAT32;
  auto promote = [](int32_t t) { return type_width(t) < 4 ? (int32_t)B2_INT32 : t; };  // bool, (u)int8, (u)int16 -> int
  a = promote(a);
  b = promote(b);
  if (a == b) return a;
  if (is_signed_id(a) == is_signed_id(b)) return type_width(a) >= type_width(b) ? a : b;
  const int32_t s = is_signed_id(a) ? a : b, u = is_signed_id(a) ? b : a;
  return type_width(u) >= type_width(s) ? u : s;  // a strictly wider signed type holds every value of the unsigned one
}

// util.cpp's rule over the numeric types (an operator is supported when it is invocable on std::common_type<lhs, rhs> and
// its result converts to `out`), and the chrono subset this library computes
bool supported(int32_t out, int32_t lhs, int32_t rhs, int32_t op)
{
  if (is_chrono(lhs) || is_chrono(rhs)) {
    if (lhs != rhs) return false;
    if (op >= B2_BINOP_EQUAL && op <= B2_BINOP_NULL_NOT_EQUALS) return out == B2_BOOL8;
    if (op == B2_BINOP_NULL_MAX || op == B2_BINOP_NULL_MIN) return out == lhs;
    return false;
  }
  if (!is_numeric(lhs) || !is_numeric(rhs) || !is_numeric(out)) return false;
  if (is_bool_op(op)) return out == B2_BOOL8;
  const int32_t c = common_type(lhs, rhs);
  if (op == B2_BINOP_SHIFT_RIGHT_UNSIGNED) return is_integral_id(c) && c != B2_BOOL8;
  if (is_integer_op(op)) return is_integral_id(c);
  return (op >= B2_BINOP_ADD && op <= B2_BINOP_ATAN2) || op == B2_BINOP_NULL_MAX || op == B2_BINOP_NULL_MIN;
}

// the kernel's compute type: C = std::common_type<out, lhs, rhs> (a chrono pair has none with BOOL8 and computes in its
// storage integers), narrowed to what C++ computes in (see binaryop.cuh)
int32_t kernel_type(int32_t op, int32_t out, int32_t lhs, int32_t rhs)
{
  int32_t c = is_chrono(lhs) ? storage_type(lhs) : common_type(common_type(out, lhs), rhs);
  if (is_integer_op(op) && is_float_id(c)) c = common_type(lhs, rhs);  // undefined values: the reference writes none
  if (op == B2_BINOP_SHIFT_RIGHT_UNSIGNED && (c == B2_INT8 || c == B2_INT16)) return c;
  return type_width(c) < 4 ? (int32_t)B2_INT32 : c;
}

void launch_family(int32_t op, int32_t ctype, const args& a, cudaStream_t stream)
{
  switch (op) {
    case B2_BINOP_ADD: case B2_BINOP_SUB: case B2_BINOP_MUL: case B2_BINOP_DIV: case B2_BINOP_FLOOR_DIV: case B2_BINOP_MOD:
    case B2_BINOP_PMOD: case B2_BINOP_PYMOD: case B2_BINOP_NULL_MAX: case B2_BINOP_NULL_MIN: return launch_arith(op, ctype, a, stream);
    case B2_BINOP_TRUE_DIV: case B2_BINOP_POW: case B2_BINOP_INT_POW: case B2_BINOP_LOG_BASE: case B2_BINOP_ATAN2:
      return launch_math(op, ctype, a, stream);
    case B2_BINOP_SHIFT_LEFT: case B2_BINOP_SHIFT_RIGHT: case B2_BINOP_SHIFT_RIGHT_UNSIGNED: case B2_BINOP_BITWISE_AND:
    case B2_BINOP_BITWISE_OR: case B2_BINOP_BITWISE_XOR: return launch_bits(op, ctype, a, stream);
    case B2_BINOP_LOGICAL_AND: case B2_BINOP_LOGICAL_OR: case B2_BINOP_NULL_LOGICAL_AND: case B2_BINOP_NULL_LOGICAL_OR:
      return launch_logical(op, ctype, a, stream);
    default: return launch_compare(op, ctype, a, stream);
  }
}

// one operand: a column view or a scalar
struct side {
  const b2_column_view* col;
  const b2_scalar* scl;
  int32_t type() const { return col ? col->type_id : scl->type_id; }
};

operand make_operand(const side& s, bool scalar_valid)
{
  operand o{};
  o.type = storage_type(s.type());
  if (s.scl) {
    o.data   = s.scl->data.ptr;
    o.scalar = true;
    o.valid  = scalar_valid;
    return o;
  }
  const b2_column_view& c = *s.col;
  o.data  = static_cast<const char*>(c.data) + (size_t)c.offset * type_width(c.type_id);
  o.mask  = has_nulls(c) ? c.null_mask : nullptr;
  o.bit   = c.offset;
  o.last_word = ((int64_t)c.offset + c.size - 1) >> 5;
  o.valid = true;
  return o;
}

bool scalar_is_valid(const b2_scalar& s, cudaStream_t stream)
{
  int32_t v = 0;
  B2_CUDA_TRY(cudaMemcpyAsync(&v, static_cast<const char*>(s.data.ptr) + 8, sizeof(v), cudaMemcpyDeviceToHost, stream));
  B2_CUDA_TRY(cudaStreamSynchronize(stream));
  return v != 0;
}

bool aligned16(const operand& o) { return o.scalar || (reinterpret_cast<uintptr_t>(o.data) & 15) == 0; }

column_ptr binary_operation(const side& l, const side& r, int32_t op, int32_t out_type, cudaStream_t stream)
{
  if (l.col && r.col) B2_EXPECTS(l.col->size == r.col->size, B2_ERR_INVALID_ARGUMENT, "Column sizes don't match");
  for (int32_t t : {l.type(), r.type(), out_type}) B2_EXPECTS(t >= 0 && t < NUM_TYPE_IDS, B2_ERR_LOGIC, "Invalid type_id");
  B2_EXPECTS(supported(out_type, l.type(), r.type(), op), B2_ERR_DATA_TYPE, "Unsupported operator for these types");
  if (l.col) validate_column(*l.col);
  if (r.col) validate_column(*r.col);
  const int32_t n = l.col ? l.col->size : r.col->size;
  if (n == 0) return make_column(out_type, 0, false, stream);

  const bool lvalid = l.scl ? scalar_is_valid(*l.scl, stream) : true;
  const bool rvalid = r.scl ? scalar_is_valid(*r.scl, stream) : true;
  const bool aware  = is_null_aware(op);
  if (!aware && !(lvalid && rvalid)) {  // a null scalar: every row null (make_column zeroes the mask)
    auto out = make_column(out_type, n, true, stream);
    out->null_count = n;
    B2_CUDA_TRY(cudaMemsetAsync(out->data.ptr, 0, out->data.bytes, stream));
    return out;
  }
  const bool with_mask = aware || (l.col && has_nulls(*l.col)) || (r.col && has_nulls(*r.col));
  auto out = make_column(out_type, n, with_mask, stream);
  if (with_mask) {
    out->pending        = dbuf(sizeof(unsigned long long), stream);
    out->pending_stream = stream;
    out->null_count     = -1;
    B2_CUDA_TRY(cudaMemsetAsync(out->pending.ptr, 0, sizeof(unsigned long long), stream));
  }
  args a{};
  a.a = make_operand(l, lvalid);
  a.b = make_operand(r, rvalid);
  a.o = result{out->data.ptr, with_mask ? out->mask.as<uint32_t>() : nullptr, storage_type(out_type),
               with_mask ? out->pending.as<unsigned long long>() : nullptr};
  a.n = n;
  const int32_t ct = kernel_type(op, out_type, l.type(), r.type());
  a.fast = !aware && a.a.type == ct && a.b.type == ct && a.o.type == (is_bool_op(op) ? (int32_t)B2_BOOL8 : ct) && aligned16(a.a) &&
           aligned16(a.b);
  prof_scope ps("binary_operation", stream);
  launch_family(op, ct, a, stream);
  return out;
}

}  // namespace
}  // namespace b2

using namespace b2;

extern "C" {

b2_status b2_binary_operation(const b2_column_view* lhs, const b2_column_view* rhs, int32_t op, int32_t out_type, b2_stream stream,
                              b2_column** out)
{
  B2_TRY_BEGIN
  B2_EXPECTS(lhs && rhs && out, B2_ERR_INVALID_ARGUMENT, "null argument");
  *out = binary_operation(side{lhs, nullptr}, side{rhs, nullptr}, op, out_type, static_cast<cudaStream_t>(stream)).release();
  B2_TRY_END
}

b2_status b2_binary_operation_cs(const b2_column_view* lhs, const b2_scalar* rhs, int32_t op, int32_t out_type, b2_stream stream,
                                 b2_column** out)
{
  B2_TRY_BEGIN
  B2_EXPECTS(lhs && rhs && out, B2_ERR_INVALID_ARGUMENT, "null argument");
  *out = binary_operation(side{lhs, nullptr}, side{nullptr, rhs}, op, out_type, static_cast<cudaStream_t>(stream)).release();
  B2_TRY_END
}

b2_status b2_binary_operation_sc(const b2_scalar* lhs, const b2_column_view* rhs, int32_t op, int32_t out_type, b2_stream stream,
                                 b2_column** out)
{
  B2_TRY_BEGIN
  B2_EXPECTS(lhs && rhs && out, B2_ERR_INVALID_ARGUMENT, "null argument");
  *out = binary_operation(side{nullptr, lhs}, side{rhs, nullptr}, op, out_type, static_cast<cudaStream_t>(stream)).release();
  B2_TRY_END
}

b2_status b2_binary_is_supported_operation(int32_t out_type, int32_t lhs_type, int32_t rhs_type, int32_t op, int32_t* result)
{
  B2_TRY_BEGIN
  B2_EXPECTS(result, B2_ERR_INVALID_ARGUMENT, "null argument");
  for (int32_t t : {lhs_type, rhs_type, out_type}) B2_EXPECTS(t >= 0 && t < NUM_TYPE_IDS, B2_ERR_LOGIC, "Invalid type_id");
  *result = supported(out_type, lhs_type, rhs_type, op) ? 1 : 0;
  B2_TRY_END
}

}  // extern "C"
