// replace.cu — cudf::replace_nulls (column, scalar, preceding / following fill), replace_nans, find_and_replace_all, clamp and
// normalize_nans_and_zeros over fixed-width columns (cpp/include/cudf/replace.hpp and cpp/src/replace/{nulls,nans,replace,
// clamp}.cu of the reference): the checks, the output column and one launch of replace_kernel or fill_kernel (replace.cuh).
//
// Unlike the reference, one kernel writes the values, the mask and the null count of every form: the fill is one look-back
// pass instead of a scan that writes a row map and a gather, and find_and_replace_all searches a sorted table of the old
// values instead of scanning all of them for every row. The null count goes into the column's pending counter; the only
// read-backs are scalars' validity where it decides the shape of the output (replace_nulls with a scalar, clamp).
#include "replace.cuh"

namespace b2 {
namespace {

using namespace repl;

// f(T{}) with the kernel type of a storage type id (BOOL8 as uint8)
template <typename F>
void with_type(int32_t sid, F&& f)
{
  switch (sid) {
    case B2_INT8: return f(int8_t{});
    case B2_INT16: return f(int16_t{});
    case B2_INT32: return f(int32_t{});
    case B2_INT64: return f(int64_t{});
    case B2_UINT8: case B2_BOOL8: return f(uint8_t{});
    case B2_UINT16: return f(uint16_t{});
    case B2_UINT32: return f(uint32_t{});
    case B2_UINT64: return f(uint64_t{});
    case B2_FLOAT32: return f(float{});
    case B2_FLOAT64: return f(double{});
    default: B2_FAIL(B2_ERR_DATA_TYPE, "replace: unsupported column type");
  }
}

const void* row0(const b2_column_view& c) { return static_cast<const char*>(c.data) + (size_t)c.offset * type_width(c.type_id); }

side column_side(const b2_column_view& c)
{
  side s{};
  s.data      = row0(c);
  s.mask      = has_nulls(c) ? c.null_mask : nullptr;
  s.bit       = c.offset;
  s.last_word = ((int64_t)c.offset + c.size - 1) >> 5;
  return s;
}

side scalar_side(const b2_scalar& s)
{
  side r{};
  r.data         = s.data.ptr;
  r.scalar_valid = reinterpret_cast<const int32_t*>(static_cast<const char*>(s.data.ptr) + 8);
  return r;
}

bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

// a copy of the view: its values, its mask realigned to offset 0 (when it has one) and its null count
column_ptr copy_of(const b2_column_view& c, cudaStream_t stream)
{
  auto out = make_column(c.type_id, c.size, false, stream);
  if (c.size == 0) return out;
  B2_CUDA_TRY(cudaMemcpyAsync(out->data.ptr, row0(c), (size_t)c.size * type_width(c.type_id), cudaMemcpyDeviceToDevice, stream));
  if (c.null_mask) {
    out->mask       = copy_bitmask(c.null_mask, c.offset, (int64_t)c.offset + c.size, stream);
    out->null_count = c.null_count;
  }
  return out;
}

// an output with a mask whose null count the kernel accumulates
unsigned long long* count_nulls(b2_column& out, cudaStream_t stream)
{
  out.pending        = dbuf(sizeof(unsigned long long), stream);
  out.pending_stream = stream;
  out.null_count     = -1;
  B2_CUDA_TRY(cudaMemsetAsync(out.pending.ptr, 0, sizeof(unsigned long long), stream));
  return out.pending.as<unsigned long long>();
}

args make_args(const b2_column_view& in, b2_column& out)
{
  args a{};
  a.in       = column_side(in);
  a.out      = out.data.ptr;
  a.out_mask = out.mask.as<uint32_t>();
  a.n        = in.size;
  a.fast     = aligned16(a.in.data) && aligned16(a.out);
  return a;
}

void read_validity(std::initializer_list<std::pair<const b2_scalar*, int32_t*>> scalars, cudaStream_t stream)
{
  for (auto& [s, v] : scalars)
    B2_CUDA_TRY(cudaMemcpyAsync(v, static_cast<const char*>(s->data.ptr) + 8, sizeof(int32_t), cudaMemcpyDeviceToHost, stream));
  B2_CUDA_TRY(cudaStreamSynchronize(stream));
}

void launch_nulls(const args& a, int width, cudaStream_t stream)
{
  prof_scope ps("replace_nulls", stream);
  dispatch_width(width, [&](auto u) { launch<NULLS, decltype(u)>(a, 0, stream); });
}

column_ptr replace_nulls(const b2_column_view& in, const b2_column_view& r, cudaStream_t stream)
{
  B2_EXPECTS(in.type_id == r.type_id, B2_ERR_DATA_TYPE, "Data type mismatch");
  B2_EXPECTS(in.size == r.size, B2_ERR_LOGIC, "Column size mismatch");
  validate_column(in);
  validate_column(r);
  if (in.size == 0) return make_column(in.type_id, 0, false, stream);
  if (!has_nulls(in)) return copy_of(in, stream);
  const bool with_mask = has_nulls(r);
  auto out = make_column(in.type_id, in.size, with_mask, stream);
  args a   = make_args(in, *out);
  a.repl   = column_side(r);
  a.fast   = a.fast && aligned16(a.repl.data);
  if (with_mask) a.nulls = count_nulls(*out, stream);
  launch_nulls(a, type_width(in.type_id), stream);
  return out;
}

column_ptr replace_nulls(const b2_column_view& in, const b2_scalar& s, cudaStream_t stream)
{
  validate_column(in);
  if (in.size == 0) return make_column(in.type_id, 0, false, stream);
  if (!has_nulls(in)) return copy_of(in, stream);
  int32_t valid = 0;
  read_validity({{&s, &valid}}, stream);
  if (!valid) return copy_of(in, stream);
  B2_EXPECTS(in.type_id == s.type_id, B2_ERR_DATA_TYPE, "Data type mismatch");
  auto out = make_column(in.type_id, in.size, false, stream);
  args a   = make_args(in, *out);
  a.repl   = scalar_side(s);
  launch_nulls(a, type_width(in.type_id), stream);
  return out;
}

column_ptr replace_nulls(const b2_column_view& in, int32_t policy, cudaStream_t stream)
{
  B2_EXPECTS(policy == B2_REPLACE_PRECEDING || policy == B2_REPLACE_FOLLOWING, B2_ERR_LOGIC, "Invalid replace_policy");
  validate_column(in);
  if (in.size == 0) return make_column(in.type_id, 0, false, stream);
  if (!has_nulls(in)) return copy_of(in, stream);
  auto out = make_column(in.type_id, in.size, true, stream);
  fill_args f{};
  f.in        = row0(in);
  f.mask      = in.null_mask;
  f.bit       = in.offset;
  f.last_word = ((int64_t)in.offset + in.size - 1) >> 5;
  f.out       = out->data.ptr;
  f.out_mask  = out->mask.as<uint32_t>();
  f.nulls     = count_nulls(*out, stream);
  f.n         = in.size;
  const int64_t ntiles = (f.n + FL_TILE - 1) / FL_TILE;
  dbuf work(sizeof(uint4) * (size_t)(ntiles + 1), stream);
  B2_CUDA_TRY(cudaMemsetAsync(work.ptr, 0, work.bytes, stream));
  scan_state st;
  st.rec    = work.as<uint4>();
  st.ticket = reinterpret_cast<uint32_t*>(work.as<uint4>() + ntiles);
  prof_scope ps("replace_nulls_policy", stream);
  dispatch_width(type_width(in.type_id), [&](auto u) {
    using T = decltype(u);
    if (policy == B2_REPLACE_PRECEDING) B2_LAUNCH((fill_kernel<T, false>), (unsigned)ntiles, FL_THREADS, 0, stream, f, st, ntiles);
    else B2_LAUNCH((fill_kernel<T, true>), (unsigned)ntiles, FL_THREADS, 0, stream, f, st, ntiles);
  });
  return out;
}

// replace_nans: FLOAT32 / FLOAT64; the output has a mask when the input has nulls or the replacement may (copy_if_else's rule)
column_ptr replace_nans(const b2_column_view& in, const side& r, int32_t r_type, bool r_nullable, cudaStream_t stream)
{
  validate_column(in);
  B2_EXPECTS(is_float_id(in.type_id), B2_ERR_LOGIC, "NAN is not supported in a Non-floating point type column");
  B2_EXPECTS(in.type_id == r_type, B2_ERR_LOGIC, "Input and replacement must be of the same type");
  if (in.size == 0) return make_column(in.type_id, 0, false, stream);
  const bool with_mask = has_nulls(in) || r_nullable;
  auto out = make_column(in.type_id, in.size, with_mask, stream);
  args a   = make_args(in, *out);
  a.repl   = r;
  a.fast   = a.fast && (r.scalar_valid || aligned16(r.data));
  if (with_mask) a.nulls = count_nulls(*out, stream);
  prof_scope ps("replace_nans", stream);
  if (in.type_id == B2_FLOAT32) launch<NANS, float>(a, 0, stream);
  else launch<NANS, double>(a, 0, stream);
  return out;
}

column_ptr find_and_replace_all(const b2_column_view& in, const b2_column_view& old, const b2_column_view& neu, cudaStream_t stream)
{
  B2_EXPECTS(old.size == neu.size, B2_ERR_LOGIC, "values_to_replace and replacement_values size mismatch.");
  B2_EXPECTS(in.type_id == old.type_id && in.type_id == neu.type_id, B2_ERR_DATA_TYPE, "Columns type mismatch");
  validate_column(in);
  validate_column(old);
  validate_column(neu);
  B2_EXPECTS(!has_nulls(old), B2_ERR_LOGIC, "values_to_replace must not have nulls");
  if (in.size == 0 || old.size == 0) return copy_of(in, stream);

  // the table: the old values' keys in a stable order of their bit patterns, each with its position
  const int w  = type_width(in.type_id);
  const int32_t k = old.size;
  const int32_t key_type = w == 1 ? B2_UINT8 : w == 2 ? B2_UINT16 : w == 4 ? B2_UINT32 : B2_UINT64;
  auto keys = make_column(key_type, k, false, stream);
  const unsigned kgrid = (unsigned)((k + 255) / 256);
  with_type(storage_type(in.type_id), [&](auto v) {
    using T = decltype(v);
    if constexpr (std::is_floating_point_v<T>)
      B2_LAUNCH((lookup_keys_kernel<T>), kgrid, 256, 0, stream, static_cast<const T*>(row0(old)), k, keys->data.as<bits_t<T>>());
    else B2_LAUNCH((lookup_keys_kernel<bits_t<T>>), kgrid, 256, 0, stream, static_cast<const bits_t<T>*>(row0(old)), k,
                   keys->data.as<bits_t<T>>());
  });
  auto order = sorted_order({keys->view()}, std::vector<uint8_t>{(uint8_t)B2_ASCENDING}, {}, true, stream);
  // the keys first, then the positions at a 16-byte boundary: each array aligned to its element
  const size_t keys_bytes = ((size_t)w * k + 15) / 16 * 16;
  dbuf table(keys_bytes + sizeof(int32_t) * (size_t)k, stream);
  void* sorted = table.ptr;
  int32_t* pos = reinterpret_cast<int32_t*>(static_cast<char*>(table.ptr) + keys_bytes);
  dispatch_width(w, [&](auto u) {
    using U = decltype(u);
    B2_LAUNCH((lookup_table_kernel<U>), kgrid, 256, 0, stream, keys->data.as<U>(), order->data.as<int32_t>(), k, static_cast<U*>(sorted),
              pos);
  });

  const bool with_mask = has_nulls(in) || has_nulls(neu);
  auto out = make_column(in.type_id, in.size, with_mask, stream);
  args a   = make_args(in, *out);
  a.repl   = column_side(neu);
  a.keys   = sorted;
  a.pos    = pos;
  a.k      = k;
  const size_t smem = lookup_smem_bytes(k, w);
  a.staged = smem <= LOOKUP_SMEM;
  if (with_mask) a.nulls = count_nulls(*out, stream);
  prof_scope ps("find_and_replace_all", stream);
  with_type(storage_type(in.type_id), [&](auto v) {
    using T = decltype(v);
    using K = std::conditional_t<std::is_floating_point_v<T>, T, bits_t<T>>;  // integers compare as their bits
    launch<LOOKUP, K>(a, a.staged ? smem : 0, stream);
  });
  return out;
}

column_ptr clamp(const b2_column_view& in, const b2_scalar& lo, const b2_scalar& lo_r, const b2_scalar& hi, const b2_scalar& hi_r,
                 cudaStream_t stream)
{
  B2_EXPECTS(lo.type_id == hi.type_id, B2_ERR_DATA_TYPE, "mismatching types of limit scalars");
  B2_EXPECTS(lo_r.type_id == hi_r.type_id, B2_ERR_DATA_TYPE, "mismatching types of replace scalars");
  B2_EXPECTS(lo.type_id == lo_r.type_id, B2_ERR_DATA_TYPE, "mismatching types of limit and replace scalars");
  validate_column(in);
  int32_t v[4] = {0, 0, 0, 0};
  read_validity({{&lo, &v[0]}, {&lo_r, &v[1]}, {&hi, &v[2]}, {&hi_r, &v[3]}}, stream);
  if ((!v[0] && !v[2]) || in.size == 0) return copy_of(in, stream);
  if (v[0]) B2_EXPECTS(v[1], B2_ERR_LOGIC, "lo_replace can't be null if lo is not null");
  if (v[2]) B2_EXPECTS(v[3], B2_ERR_LOGIC, "hi_replace can't be null if hi is not null");
  B2_EXPECTS(in.type_id == lo.type_id, B2_ERR_DATA_TYPE, "mismatching types of scalar and input");

  auto out = make_column(in.type_id, in.size, in.null_mask != nullptr, stream);  // the input's mask and null count
  out->null_count = in.null_mask ? in.null_count : 0;
  args a = make_args(in, *out);
  a.lo   = v[0] ? lo.data.ptr : nullptr;
  a.lo_r = v[0] ? lo_r.data.ptr : nullptr;
  a.hi   = v[2] ? hi.data.ptr : nullptr;
  a.hi_r = v[2] ? hi_r.data.ptr : nullptr;
  if (!in.null_mask) a.out_mask = nullptr;
  prof_scope ps("clamp", stream);
  with_type(storage_type(in.type_id), [&](auto t) { launch<CLAMP, decltype(t)>(a, 0, stream); });
  return out;
}

void normalize(const args& a, int32_t type_id, cudaStream_t stream)
{
  prof_scope ps("normalize_nans_and_zeros", stream);
  if (type_id == B2_FLOAT32) launch<NORMALIZE, float>(a, 0, stream);
  else launch<NORMALIZE, double>(a, 0, stream);
}

column_ptr normalize_nans_and_zeros(const b2_column_view& in, cudaStream_t stream)
{
  validate_column(in);
  if (in.size == 0) return copy_of(in, stream);
  B2_EXPECTS(is_float_id(in.type_id), B2_ERR_LOGIC, "Expects float or double input");
  auto out = make_column(in.type_id, in.size, in.null_mask != nullptr, stream);
  out->null_count = in.null_mask ? in.null_count : 0;
  normalize(make_args(in, *out), in.type_id, stream);
  return out;
}

void normalize_nans_and_zeros_inplace(const b2_column_view& c, cudaStream_t stream)
{
  validate_column(c);
  if (c.size == 0) return;
  B2_EXPECTS(is_float_id(c.type_id), B2_ERR_LOGIC, "Expects float or double input");
  args a{};
  a.in   = column_side(c);
  a.out  = const_cast<void*>(a.in.data);
  a.n    = c.size;
  a.fast = false;  // the vector path reads through the non-coherent cache, which a kernel writing the same data must not use
  normalize(a, c.type_id, stream);
}

}  // namespace
}  // namespace b2

using namespace b2;

extern "C" {

b2_status b2_replace_nulls(const b2_column_view* input, const b2_column_view* replacement, b2_stream stream, b2_column** out)
{
  B2_TRY_BEGIN
  B2_EXPECTS(input && replacement && out, B2_ERR_INVALID_ARGUMENT, "null argument");
  *out = replace_nulls(*input, *replacement, static_cast<cudaStream_t>(stream)).release();
  B2_TRY_END
}

b2_status b2_replace_nulls_scalar(const b2_column_view* input, const b2_scalar* replacement, b2_stream stream, b2_column** out)
{
  B2_TRY_BEGIN
  B2_EXPECTS(input && replacement && out, B2_ERR_INVALID_ARGUMENT, "null argument");
  *out = replace_nulls(*input, *replacement, static_cast<cudaStream_t>(stream)).release();
  B2_TRY_END
}

b2_status b2_replace_nulls_policy(const b2_column_view* input, int32_t policy, b2_stream stream, b2_column** out)
{
  B2_TRY_BEGIN
  B2_EXPECTS(input && out, B2_ERR_INVALID_ARGUMENT, "null argument");
  *out = replace_nulls(*input, policy, static_cast<cudaStream_t>(stream)).release();
  B2_TRY_END
}

b2_status b2_replace_nans(const b2_column_view* input, const b2_column_view* replacement, b2_stream stream, b2_column** out)
{
  B2_TRY_BEGIN
  B2_EXPECTS(input && replacement && out, B2_ERR_INVALID_ARGUMENT, "null argument");
  B2_EXPECTS(input->size == replacement->size, B2_ERR_LOGIC, "Input and replacement must be of the same size");
  validate_column(*replacement);
  side r{};
  if (replacement->size) r = column_side(*replacement);
  *out = replace_nans(*input, r, replacement->type_id, replacement->null_mask != nullptr, static_cast<cudaStream_t>(stream)).release();
  B2_TRY_END
}

b2_status b2_replace_nans_scalar(const b2_column_view* input, const b2_scalar* replacement, b2_stream stream, b2_column** out)
{
  B2_TRY_BEGIN
  B2_EXPECTS(input && replacement && out, B2_ERR_INVALID_ARGUMENT, "null argument");
  *out = replace_nans(*input, scalar_side(*replacement), replacement->type_id, true, static_cast<cudaStream_t>(stream)).release();
  B2_TRY_END
}

b2_status b2_find_and_replace_all(const b2_column_view* input, const b2_column_view* values_to_replace,
                                  const b2_column_view* replacement_values, b2_stream stream, b2_column** out)
{
  B2_TRY_BEGIN
  B2_EXPECTS(input && values_to_replace && replacement_values && out, B2_ERR_INVALID_ARGUMENT, "null argument");
  *out = find_and_replace_all(*input, *values_to_replace, *replacement_values, static_cast<cudaStream_t>(stream)).release();
  B2_TRY_END
}

b2_status b2_clamp(const b2_column_view* input, const b2_scalar* lo, const b2_scalar* lo_replace, const b2_scalar* hi,
                   const b2_scalar* hi_replace, b2_stream stream, b2_column** out)
{
  B2_TRY_BEGIN
  B2_EXPECTS(input && lo && lo_replace && hi && hi_replace && out, B2_ERR_INVALID_ARGUMENT, "null argument");
  *out = b2::clamp(*input, *lo, *lo_replace, *hi, *hi_replace, static_cast<cudaStream_t>(stream)).release();
  B2_TRY_END
}

b2_status b2_normalize_nans_and_zeros(const b2_column_view* input, b2_stream stream, b2_column** out)
{
  B2_TRY_BEGIN
  B2_EXPECTS(input && out, B2_ERR_INVALID_ARGUMENT, "null argument");
  *out = normalize_nans_and_zeros(*input, static_cast<cudaStream_t>(stream)).release();
  B2_TRY_END
}

b2_status b2_normalize_nans_and_zeros_inplace(const b2_column_view* in_out, b2_stream stream)
{
  B2_TRY_BEGIN
  B2_EXPECTS(in_out, B2_ERR_INVALID_ARGUMENT, "null argument");
  normalize_nans_and_zeros_inplace(*in_out, static_cast<cudaStream_t>(stream));
  B2_TRY_END
}

}  // extern "C"
