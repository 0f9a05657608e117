// unary.cu — cudf::unary_operation, cast, is_supported_cast, is_null / is_valid and is_nan / is_not_nan over fixed-width columns
// (cpp/include/cudf/unary.hpp and cpp/src/unary/{math_ops,cast_ops,nan_ops,null_ops}.cu of the reference): the type rules, the
// checks, the output column and one launch of a family's kernel (unary.cuh).
//
// Unlike the reference (copy_bitmask, then a transform) one kernel writes the values and the output mask words; the null count
// is the input's. No call synchronises.
#include "unary.cuh"

namespace b2 {
namespace {

using namespace unary;

constexpr int32_t NUM_TYPE_IDS = 29;  // cudf::type_id::NUM_TYPE_IDS
constexpr int32_t DECIMAL32 = 25, DECIMAL128 = 27;

bool is_timestamp(int32_t id) { return id >= B2_TIMESTAMP_DAYS && id <= B2_TIMESTAMP_NANOSECONDS; }
bool is_duration(int32_t id) { return id >= B2_DURATION_DAYS && id <= B2_DURATION_NANOSECONDS; }
bool is_decimal(int32_t id) { return id >= DECIMAL32 && id <= DECIMAL128; }

// math_ops.cu's dispatchers: the output type of `op` on `t`, or -1 when the pair has no kernel there
int32_t op_output(int32_t op, int32_t t)
{
  const bool arith = is_numeric(t), integral = is_integral_id(t);
  if (op >= B2_UNARY_SIN && op <= B2_UNARY_ABS) return arith ? t : -1;
  switch (op) {
    case B2_UNARY_RINT: return is_float_id(t) ? t : -1;
    case B2_UNARY_BIT_COUNT: return integral ? (int32_t)B2_INT32 : -1;
    case B2_UNARY_BIT_INVERT: return integral ? t : -1;
    case B2_UNARY_NOT: return arith ? (int32_t)B2_BOOL8 : -1;
    case B2_UNARY_NEGATE: return (is_signed_id(t) || is_float_id(t) || is_duration(t)) ? t : -1;
    default: return -1;
  }
}

// cast_ops.cu's is_supported_non_fixed_point_cast over the ids this library holds; a decimal pair is not supported here
bool cast_supported(int32_t from, int32_t to)
{
  if (!is_fixed_width(from) || !is_fixed_width(to)) return false;
  return !(is_timestamp(from) && is_numeric(to)) && !(is_numeric(from) && is_timestamp(to));
}

// ticks per day of a chrono id
int64_t ticks_per_day(int32_t id)
{
  switch ((id - B2_TIMESTAMP_DAYS) % 5) {
    case 0: return 1;
    case 1: return 86400LL;
    case 2: return 86400LL * 1000;
    case 3: return 86400LL * 1000000;
    default: return 86400LL * 1000000000;
  }
}

args make_args(const b2_column_view& c, void* out, uint32_t* out_mask, int32_t out_type)
{
  args a{};
  a.in        = static_cast<const char*>(c.data) + (size_t)c.offset * type_width(c.type_id);
  a.mask      = c.null_mask;
  a.bit       = c.offset;
  a.last_word = ((int64_t)c.offset + c.size - 1) >> 5;
  a.in_type   = storage_type(c.type_id);
  a.out_type  = storage_type(out_type);
  a.out       = out;
  a.out_mask  = out_mask;
  a.n         = c.size;
  a.fold      = -1;
  a.fast      = (reinterpret_cast<uintptr_t>(a.in) & 15) == 0 && (reinterpret_cast<uintptr_t>(out) & 15) == 0;
  return a;
}

// the output column of an elementwise pass: a mask exactly when the input has one, and the input's null count
column_ptr output_like(const b2_column_view& c, int32_t out_type, cudaStream_t stream)
{
  const bool with_mask = c.null_mask != nullptr;
  auto out             = make_column(out_type, c.size, with_mask, stream);
  if (with_mask) out->null_count = c.null_count;
  return out;
}

void check_type_id(int32_t t) { B2_EXPECTS(t >= 0 && t < NUM_TYPE_IDS, B2_ERR_LOGIC, "Invalid type_id"); }

column_ptr unary_operation(const b2_column_view& c, int32_t op, cudaStream_t stream)
{
  B2_EXPECTS(op >= B2_UNARY_SIN && op <= B2_UNARY_NEGATE, B2_ERR_LOGIC, "Undefined unary operation");
  validate_column(c);
  if (c.size == 0) {
    const int32_t t = op == B2_UNARY_NOT ? (int32_t)B2_BOOL8 : op == B2_UNARY_BIT_COUNT ? (int32_t)B2_INT32 : c.type_id;
    return make_column(t, 0, false, stream);
  }
  const int32_t t = op_output(op, c.type_id);
  B2_EXPECTS(t >= 0, B2_ERR_LOGIC, "Unsupported data type for this unary operation");
  auto out = output_like(c, t, stream);
  const args a = make_args(c, out->data.ptr, out->mask.as<uint32_t>(), t);
  prof_scope ps("unary_operation", stream);
  if (op <= B2_UNARY_RINT) launch_math(op, a, stream);
  else launch_bits(op, a, stream);
  return out;
}

column_ptr cast(const b2_column_view& c, int32_t to, cudaStream_t stream)
{
  check_type_id(to);
  B2_EXPECTS(!is_decimal(to), B2_ERR_DATA_TYPE, "cast: decimal types are not supported");
  B2_EXPECTS(is_fixed_width(to), B2_ERR_LOGIC, "Unary cast type must be fixed-width.");
  validate_column(c);
  const int32_t from = c.type_id;
  B2_EXPECTS(cast_supported(from, to), B2_ERR_LOGIC, "Unsupported cast between a timestamp and a numeric type");
  auto out = output_like(c, to, stream);
  if (c.size == 0) return out;

  const bool chrono = (is_timestamp(from) || is_duration(from)) && (is_timestamp(to) || is_duration(to));
  int64_t mul = 1, div = 1;
  if (chrono) {
    const int64_t f = ticks_per_day(from), t = ticks_per_day(to);
    if (t >= f) mul = t / f;
    else div = f / t;
  }
  if (storage_type(from) == storage_type(to) && mul == 1 && div == 1) {  // the same values: a copy
    const size_t w = type_width(from);
    B2_CUDA_TRY(cudaMemcpyAsync(out->data.ptr, static_cast<const char*>(c.data) + (size_t)c.offset * w, (size_t)c.size * w,
                                cudaMemcpyDeviceToDevice, stream));
    if (c.null_mask) out->mask = copy_bitmask(c.null_mask, c.offset, (int64_t)c.offset + c.size, stream);
    return out;
  }
  args a = make_args(c, out->data.ptr, out->mask.as<uint32_t>(), to);
  if (chrono) {
    a.mul = mul;
    a.div = div;
  }
  prof_scope ps("cast", stream);
  launch_cast(a, stream);
  return out;
}

column_ptr is_nan(const b2_column_view& c, bool want_nan, cudaStream_t stream)
{
  validate_column(c);
  B2_EXPECTS(is_float_id(c.type_id), B2_ERR_LOGIC, "NAN is not supported in a Non-floating point type column");
  auto out = make_column(B2_BOOL8, c.size, false, stream);
  if (c.size == 0) return out;
  args a = make_args(c, out->data.ptr, nullptr, B2_BOOL8);
  if (!has_nulls(c)) a.mask = nullptr;
  a.fold = want_nan ? 0 : 1;
  prof_scope ps("is_nan", stream);
  launch_nan(want_nan, a, stream);
  return out;
}

column_ptr is_valid(const b2_column_view& c, bool want_valid, cudaStream_t stream)
{
  validate_column(c);
  auto out = make_column(B2_BOOL8, c.size, false, stream);
  if (c.size == 0) return out;
  if (!has_nulls(c) || c.null_count == c.size) {  // every row valid, or every row null: a constant
    const bool all_valid = !has_nulls(c);
    B2_CUDA_TRY(cudaMemsetAsync(out->data.ptr, all_valid == want_valid ? 1 : 0, (size_t)c.size, stream));
    return out;
  }
  const args a = make_args(c, out->data.ptr, nullptr, B2_BOOL8);
  prof_scope ps("is_null", stream);
  launch_validity(want_valid, a, stream);
  return out;
}

}  // namespace
}  // namespace b2

using namespace b2;

extern "C" {

b2_status b2_unary_operation(const b2_column_view* input, int32_t op, b2_stream stream, b2_column** out)
{
  B2_TRY_BEGIN
  B2_EXPECTS(input && out, B2_ERR_INVALID_ARGUMENT, "null argument");
  *out = unary_operation(*input, op, static_cast<cudaStream_t>(stream)).release();
  B2_TRY_END
}

b2_status b2_cast(const b2_column_view* input, int32_t out_type, b2_stream stream, b2_column** out)
{
  B2_TRY_BEGIN
  B2_EXPECTS(input && out, B2_ERR_INVALID_ARGUMENT, "null argument");
  *out = b2::cast(*input, out_type, static_cast<cudaStream_t>(stream)).release();
  B2_TRY_END
}

b2_status b2_is_supported_cast(int32_t from_type, int32_t to_type, int32_t* result)
{
  B2_TRY_BEGIN
  B2_EXPECTS(result, B2_ERR_INVALID_ARGUMENT, "null argument");
  check_type_id(from_type);
  check_type_id(to_type);
  *result = cast_supported(from_type, to_type) ? 1 : 0;
  B2_TRY_END
}

b2_status b2_is_null(const b2_column_view* input, b2_stream stream, b2_column** out)
{
  B2_TRY_BEGIN
  B2_EXPECTS(input && out, B2_ERR_INVALID_ARGUMENT, "null argument");
  *out = is_valid(*input, false, static_cast<cudaStream_t>(stream)).release();
  B2_TRY_END
}

b2_status b2_is_valid(const b2_column_view* input, b2_stream stream, b2_column** out)
{
  B2_TRY_BEGIN
  B2_EXPECTS(input && out, B2_ERR_INVALID_ARGUMENT, "null argument");
  *out = is_valid(*input, true, static_cast<cudaStream_t>(stream)).release();
  B2_TRY_END
}

b2_status b2_is_nan(const b2_column_view* input, b2_stream stream, b2_column** out)
{
  B2_TRY_BEGIN
  B2_EXPECTS(input && out, B2_ERR_INVALID_ARGUMENT, "null argument");
  *out = is_nan(*input, true, static_cast<cudaStream_t>(stream)).release();
  B2_TRY_END
}

b2_status b2_is_not_nan(const b2_column_view* input, b2_stream stream, b2_column** out)
{
  B2_TRY_BEGIN
  B2_EXPECTS(input && out, B2_ERR_INVALID_ARGUMENT, "null argument");
  *out = is_nan(*input, false, static_cast<cudaStream_t>(stream)).release();
  B2_TRY_END
}

}  // extern "C"
