// b2_bridge.hpp — the libcudf C++ API surface of the hot path as header-only wrappers over the C ABI
// (include/cudf_b200.h).  Names, argument order and defaults follow the reference headers:
//   cudf/types.hpp:76-340, column/column_view.hpp:44-245, column/column.hpp:36-334,
//   table/table_view.hpp:41-206, table/table.hpp:31-215, sorting.hpp:44-163, copying.hpp:37-126,
//   join/join.hpp:72-249, join/hash_join.hpp, groupby.hpp:54-184, aggregation.hpp:78-266,
//   reduction.hpp, null_mask.hpp, utilities/error.hpp:35-118.
// rmm:: types are minimal stand-ins so that reference call sites compile unchanged; `mr` arguments are
// accepted and ignored (device memory comes from the library's stream-ordered pool).
#pragma once

#include "../../cudf_b200.h"

#include <cstddef>
#include <cstdint>
#include <memory>
#include <new>
#include <optional>
#include <stdexcept>
#include <string>
#include <utility>
#include <vector>

// ------------------------------------------------------------------------------------------------
// rmm stand-ins
// ------------------------------------------------------------------------------------------------
namespace rmm {
class cuda_stream_view {
 public:
  constexpr cuda_stream_view() = default;
  constexpr cuda_stream_view(void* s) : s_(s) {}
  [[nodiscard]] constexpr void* value() const noexcept { return s_; }
 private:
  void* s_{nullptr};
};
struct device_async_resource_ref {};
namespace mr { inline device_async_resource_ref get_current_device_resource_ref() { return {}; } }

template <typename T>
class device_uvector {  // owning view of an INT32/any column's data returned by the library
 public:
  device_uvector(b2_column* col, T* data, std::size_t n) : col_(col), data_(data), n_(n) {}
  device_uvector(device_uvector&& o) noexcept : col_(o.col_), data_(o.data_), n_(o.n_) { o.col_ = nullptr; }
  device_uvector(device_uvector const&) = delete;
  ~device_uvector() { if (col_) b2_column_free(col_); }
  [[nodiscard]] T* data() noexcept { return data_; }
  [[nodiscard]] T const* data() const noexcept { return data_; }
  [[nodiscard]] std::size_t size() const noexcept { return n_; }
  [[nodiscard]] bool is_empty() const noexcept { return n_ == 0; }
 private:
  b2_column* col_;
  T* data_;
  std::size_t n_;
};

class device_buffer {
 public:
  device_buffer() = default;
  explicit device_buffer(b2_buffer* b) : b_(b) {}
  device_buffer(device_buffer&& o) noexcept : b_(o.b_) { o.b_ = nullptr; }
  device_buffer& operator=(device_buffer&& o) noexcept { if (this != &o) { reset(); b_ = o.b_; o.b_ = nullptr; } return *this; }
  device_buffer(device_buffer const&) = delete;
  ~device_buffer() { reset(); }
  [[nodiscard]] void* data() const noexcept { return b_ ? b2_buffer_data(b_) : nullptr; }
  [[nodiscard]] std::size_t size() const noexcept { return b_ ? b2_buffer_size(b_) : 0; }
 private:
  void reset() { if (b_) b2_buffer_free(b_); b_ = nullptr; }
  b2_buffer* b_{nullptr};
};
}  // namespace rmm

namespace cudf {

// ------------------------------------------------------------------------------------------------
// errors (utilities/error.hpp)
// ------------------------------------------------------------------------------------------------
struct logic_error : std::logic_error { using std::logic_error::logic_error; };
struct data_type_error : std::invalid_argument { using std::invalid_argument::invalid_argument; };
struct cuda_error : std::runtime_error { using std::runtime_error::runtime_error; };

namespace detail {
inline void check(b2_status s)
{
  if (s == B2_OK) return;
  std::string const msg = b2_last_error();
  switch (s) {
    case B2_ERR_LOGIC: throw cudf::logic_error(msg);
    case B2_ERR_INVALID_ARGUMENT: throw std::invalid_argument(msg);
    case B2_ERR_DATA_TYPE: throw cudf::data_type_error(msg);
    case B2_ERR_OUT_OF_RANGE: throw std::out_of_range(msg);
    case B2_ERR_BAD_ALLOC: throw std::bad_alloc();
    default: throw cudf::cuda_error(msg);
  }
}
}  // namespace detail

// ------------------------------------------------------------------------------------------------
// types.hpp
// ------------------------------------------------------------------------------------------------
using size_type    = int32_t;
using bitmask_type = uint32_t;
enum class order : bool { ASCENDING, DESCENDING };
enum class null_policy : bool { EXCLUDE, INCLUDE };
enum class null_equality : bool { EQUAL, UNEQUAL };
enum class nan_equality : int32_t { ALL_EQUAL, UNEQUAL };  // types.hpp: NaN == NaN, or every NaN distinct
enum class null_order : bool { AFTER, BEFORE };
enum class sorted : bool { NO, YES };
enum class mask_state : int32_t { UNALLOCATED, UNINITIALIZED, ALL_VALID, ALL_NULL };
enum class out_of_bounds_policy : bool { NULLIFY, DONT_CHECK };
enum class scan_type : bool { INCLUSIVE, EXCLUSIVE };
enum class nullable_join : bool { YES, NO };
constexpr size_type JoinNoMatch = INT32_MIN;

enum class type_id : int32_t {
  EMPTY, INT8, INT16, INT32, INT64, UINT8, UINT16, UINT32, UINT64, FLOAT32, FLOAT64, BOOL8,
  TIMESTAMP_DAYS, TIMESTAMP_SECONDS, TIMESTAMP_MILLISECONDS, TIMESTAMP_MICROSECONDS, TIMESTAMP_NANOSECONDS,
  DURATION_DAYS, DURATION_SECONDS, DURATION_MILLISECONDS, DURATION_MICROSECONDS, DURATION_NANOSECONDS,
  DICTIONARY32, STRING, LIST, DECIMAL32, DECIMAL64, DECIMAL128, STRUCT, NUM_TYPE_IDS  // no column of these types exists here
};
class data_type {
 public:
  constexpr data_type() = default;
  constexpr explicit data_type(type_id id) : _id{id} {}
  [[nodiscard]] constexpr type_id id() const noexcept { return _id; }
  constexpr bool operator==(data_type const& o) const { return _id == o._id; }
 private:
  type_id _id{type_id::EMPTY};
};
template <typename T> constexpr type_id type_to_id();
template <> constexpr type_id type_to_id<int8_t>() { return type_id::INT8; }
template <> constexpr type_id type_to_id<int16_t>() { return type_id::INT16; }
template <> constexpr type_id type_to_id<int32_t>() { return type_id::INT32; }
template <> constexpr type_id type_to_id<int64_t>() { return type_id::INT64; }
template <> constexpr type_id type_to_id<uint8_t>() { return type_id::UINT8; }
template <> constexpr type_id type_to_id<uint16_t>() { return type_id::UINT16; }
template <> constexpr type_id type_to_id<uint32_t>() { return type_id::UINT32; }
template <> constexpr type_id type_to_id<uint64_t>() { return type_id::UINT64; }
template <> constexpr type_id type_to_id<float>() { return type_id::FLOAT32; }
template <> constexpr type_id type_to_id<double>() { return type_id::FLOAT64; }
template <> constexpr type_id type_to_id<bool>() { return type_id::BOOL8; }

inline rmm::cuda_stream_view get_default_stream() { return {}; }
inline rmm::device_async_resource_ref get_current_device_resource_ref() { return {}; }

// ------------------------------------------------------------------------------------------------
// column_view / table_view
// ------------------------------------------------------------------------------------------------
class column_view {
 public:
  column_view() = default;
  column_view(data_type type, size_type size, void const* data, bitmask_type const* null_mask = nullptr,
              size_type null_count = 0, size_type offset = 0)
    : v_{static_cast<int32_t>(type.id()), size, data, null_mask, null_count, offset} {}
  [[nodiscard]] data_type type() const noexcept { return data_type{static_cast<type_id>(v_.type_id)}; }
  [[nodiscard]] size_type size() const noexcept { return v_.size; }
  [[nodiscard]] bool is_empty() const noexcept { return v_.size == 0; }
  [[nodiscard]] size_type null_count() const noexcept { return v_.null_count; }
  [[nodiscard]] bool nullable() const noexcept { return v_.null_mask != nullptr; }
  [[nodiscard]] bool has_nulls() const noexcept { return v_.null_count > 0; }
  [[nodiscard]] bitmask_type const* null_mask() const noexcept { return v_.null_mask; }
  [[nodiscard]] size_type offset() const noexcept { return v_.offset; }
  template <typename T> [[nodiscard]] T const* head() const noexcept { return static_cast<T const*>(v_.data); }
  template <typename T> [[nodiscard]] T const* data() const noexcept { return head<T>() + v_.offset; }
  template <typename T> [[nodiscard]] T const* begin() const noexcept { return data<T>(); }
  template <typename T> [[nodiscard]] T const* end() const noexcept { return data<T>() + v_.size; }
  [[nodiscard]] b2_column_view const& native() const noexcept { return v_; }
 private:
  b2_column_view v_{};
};
// a view whose data the callee may write (normalize_nans_and_zeros in place); a column_view otherwise
class mutable_column_view : public column_view {
 public:
  using column_view::column_view;
  template <typename T> [[nodiscard]] T* data() const noexcept { return const_cast<T*>(column_view::data<T>()); }
};

class table_view {
 public:
  table_view() = default;
  table_view(std::vector<column_view> const& cols) : cols_(cols)
  {
    for (auto const& c : cols_)
      if (c.size() != cols_.front().size()) throw std::invalid_argument("Column size mismatch.");
  }
  [[nodiscard]] size_type num_columns() const noexcept { return static_cast<size_type>(cols_.size()); }
  [[nodiscard]] size_type num_rows() const noexcept { return cols_.empty() ? 0 : cols_.front().size(); }
  [[nodiscard]] column_view const& column(size_type i) const { return cols_.at(i); }
  [[nodiscard]] auto begin() const noexcept { return cols_.begin(); }
  [[nodiscard]] auto end() const noexcept { return cols_.end(); }
  // native view for the C ABI (valid while this object lives)
  [[nodiscard]] b2_table_view native() const
  {
    raw_.clear();
    for (auto const& c : cols_) raw_.push_back(c.native());
    return b2_table_view{raw_.data(), static_cast<int32_t>(raw_.size())};
  }
 private:
  std::vector<column_view> cols_;
  mutable std::vector<b2_column_view> raw_;
};

// ------------------------------------------------------------------------------------------------
// owning column / table / scalar
// ------------------------------------------------------------------------------------------------
class column {
 public:
  explicit column(b2_column* h) : h_(h) {}
  column(column&& o) noexcept : h_(o.h_) { o.h_ = nullptr; }
  column(column const&) = delete;
  ~column() { if (h_) b2_column_free(h_); }
  [[nodiscard]] column_view view() const
  {
    b2_column_view v{};
    detail::check(b2_column_view_of(h_, &v));
    return column_view{data_type{static_cast<type_id>(v.type_id)}, v.size, v.data, v.null_mask, v.null_count, v.offset};
  }
  operator column_view() const { return view(); }
  [[nodiscard]] mutable_column_view mutable_view()
  {
    column_view const v = view();
    return mutable_column_view{v.type(), v.size(), v.head<void>(), v.null_mask(), v.null_count(), v.offset()};
  }
  operator mutable_column_view() { return mutable_view(); }
  [[nodiscard]] data_type type() const { return view().type(); }
  [[nodiscard]] size_type size() const { return view().size(); }
  [[nodiscard]] size_type null_count() const { return view().null_count(); }
  [[nodiscard]] bool has_nulls() const { return null_count() > 0; }
  b2_column* release_handle() noexcept { auto* h = h_; h_ = nullptr; return h; }
 private:
  b2_column* h_;
};

class table {
 public:
  table() = default;
  explicit table(std::vector<std::unique_ptr<column>>&& cols) : cols_(std::move(cols)) {}
  // takes a library table handle apart (cudf::table::release semantics)
  static std::unique_ptr<table> from_handle(b2_table* t)
  {
    int32_t n = b2_table_num_columns(t);
    std::vector<b2_column*> raw(static_cast<std::size_t>(n > 0 ? n : 1));
    detail::check(b2_table_release(t, raw.data(), static_cast<int32_t>(raw.size())));
    b2_table_free(t);
    std::vector<std::unique_ptr<column>> cols;
    for (int32_t i = 0; i < n; ++i) cols.push_back(std::make_unique<column>(raw[i]));
    return std::make_unique<table>(std::move(cols));
  }
  [[nodiscard]] size_type num_columns() const noexcept { return static_cast<size_type>(cols_.size()); }
  [[nodiscard]] size_type num_rows() const { return cols_.empty() ? 0 : cols_.front()->size(); }
  [[nodiscard]] column& get_column(size_type i) { return *cols_.at(i); }
  [[nodiscard]] column const& get_column(size_type i) const { return *cols_.at(i); }
  [[nodiscard]] table_view view() const
  {
    std::vector<column_view> v;
    for (auto const& c : cols_) v.push_back(c->view());
    return table_view{v};
  }
  operator table_view() const { return view(); }
  std::vector<std::unique_ptr<column>> release() { return std::move(cols_); }
 private:
  std::vector<std::unique_ptr<column>> cols_;
};

class scalar {
 public:
  explicit scalar(b2_scalar* h) : h_(h) {}
  scalar(scalar const&) = delete;
  virtual ~scalar() { if (h_) b2_scalar_free(h_); }
  [[nodiscard]] data_type type() const { return data_type{static_cast<type_id>(b2_scalar_type(h_))}; }
  [[nodiscard]] bool is_valid(rmm::cuda_stream_view stream = get_default_stream()) const
  {
    int32_t v = 0;
    detail::check(b2_scalar_get(h_, stream.value(), nullptr, &v));
    return v != 0;
  }
  [[nodiscard]] b2_scalar const* native() const noexcept { return h_; }
 protected:
  b2_scalar* h_;
};
template <typename T>
class numeric_scalar : public scalar {
 public:
  using scalar::scalar;
  numeric_scalar(T value, bool is_valid = true, rmm::cuda_stream_view stream = get_default_stream()) : scalar(nullptr)
  {
    detail::check(b2_scalar_create(static_cast<int32_t>(type_to_id<T>()), &value, is_valid ? 1 : 0, stream.value(), &h_));
  }
  [[nodiscard]] T value(rmm::cuda_stream_view stream = get_default_stream()) const
  {
    unsigned char raw[8] = {0};
    detail::check(b2_scalar_get(h_, stream.value(), raw, nullptr));
    T out;
    __builtin_memcpy(&out, raw, sizeof(T));
    return out;
  }
};

// ------------------------------------------------------------------------------------------------
// aggregation.hpp
// ------------------------------------------------------------------------------------------------
class aggregation {
 public:
  enum Kind : int32_t { SUM = 0, PRODUCT = 2, MIN = 3, MAX = 4, COUNT_VALID = 5, COUNT_ALL = 6, SUM_OF_SQUARES = 9, MEAN = 10, M2 = 11,
                        VARIANCE = 12, STD = 13, ARGMAX = 16, ARGMIN = 17 };
  explicit aggregation(Kind k) : kind{k} {}
  virtual ~aggregation() = default;
  Kind kind;
  size_type _ddof{-1};  // VARIANCE / STD: delta degrees of freedom (aggregation.hpp:231-260); -1 = not applicable
  // the kind word of the C ABI (B2_AGG_WITH_DDOF)
  [[nodiscard]] int32_t abi_kind() const { return _ddof < 0 ? static_cast<int32_t>(kind) : B2_AGG_WITH_DDOF(kind, _ddof); }
};
class groupby_aggregation : public virtual aggregation { public: groupby_aggregation() : aggregation(SUM) {} };
class groupby_scan_aggregation : public virtual aggregation { public: groupby_scan_aggregation() : aggregation(SUM) {} };
class reduce_aggregation : public virtual aggregation { public: reduce_aggregation() : aggregation(SUM) {} };
class scan_aggregation : public virtual aggregation { public: scan_aggregation() : aggregation(SUM) {} };
class segmented_reduce_aggregation : public virtual aggregation { public: segmented_reduce_aggregation() : aggregation(SUM) {} };
namespace detail {
template <typename Base>
struct agg_impl final : Base { explicit agg_impl(aggregation::Kind k) : aggregation(k) {} };
template <typename Base> std::unique_ptr<Base> make_agg(aggregation::Kind k) { return std::make_unique<agg_impl<Base>>(k); }
}  // namespace detail
template <typename Base = aggregation> std::unique_ptr<Base> make_sum_aggregation() { return detail::make_agg<Base>(aggregation::SUM); }
template <typename Base = aggregation> std::unique_ptr<Base> make_product_aggregation() { return detail::make_agg<Base>(aggregation::PRODUCT); }
template <typename Base = aggregation> std::unique_ptr<Base> make_min_aggregation() { return detail::make_agg<Base>(aggregation::MIN); }
template <typename Base = aggregation> std::unique_ptr<Base> make_max_aggregation() { return detail::make_agg<Base>(aggregation::MAX); }
template <typename Base = aggregation> std::unique_ptr<Base> make_mean_aggregation() { return detail::make_agg<Base>(aggregation::MEAN); }
template <typename Base = aggregation> std::unique_ptr<Base> make_sum_of_squares_aggregation() { return detail::make_agg<Base>(aggregation::SUM_OF_SQUARES); }
template <typename Base = aggregation> std::unique_ptr<Base> make_m2_aggregation() { return detail::make_agg<Base>(aggregation::M2); }
template <typename Base = aggregation> std::unique_ptr<Base> make_argmax_aggregation() { return detail::make_agg<Base>(aggregation::ARGMAX); }
template <typename Base = aggregation> std::unique_ptr<Base> make_argmin_aggregation() { return detail::make_agg<Base>(aggregation::ARGMIN); }
template <typename Base = aggregation> std::unique_ptr<Base> make_variance_aggregation(size_type ddof = 1)
{
  auto a = detail::make_agg<Base>(aggregation::VARIANCE);
  a->_ddof = ddof;
  return a;
}
template <typename Base = aggregation> std::unique_ptr<Base> make_std_aggregation(size_type ddof = 1)
{
  auto a = detail::make_agg<Base>(aggregation::STD);
  a->_ddof = ddof;
  return a;
}
template <typename Base = aggregation>
std::unique_ptr<Base> make_count_aggregation(null_policy null_handling = null_policy::EXCLUDE)
{
  return detail::make_agg<Base>(null_handling == null_policy::EXCLUDE ? aggregation::COUNT_VALID : aggregation::COUNT_ALL);
}

// ------------------------------------------------------------------------------------------------
// sorting.hpp / copying.hpp
// ------------------------------------------------------------------------------------------------
namespace detail {
inline std::vector<uint8_t> u8(std::vector<order> const& v) { std::vector<uint8_t> o; for (auto x : v) o.push_back(static_cast<uint8_t>(x)); return o; }
inline std::vector<uint8_t> u8(std::vector<null_order> const& v) { std::vector<uint8_t> o; for (auto x : v) o.push_back(static_cast<uint8_t>(x)); return o; }
}  // namespace detail

#define CUDF_B2_SORT_ARGS                                                                            \
  std::vector<order> const& column_order = {}, std::vector<null_order> const& null_precedence = {},  \
  rmm::cuda_stream_view stream = cudf::get_default_stream(),                                         \
  rmm::device_async_resource_ref = cudf::get_current_device_resource_ref()

inline std::unique_ptr<column> sorted_order_impl(table_view const& input, std::vector<order> const& co,
                                                 std::vector<null_order> const& np, bool stable, rmm::cuda_stream_view stream)
{
  auto o = detail::u8(co); auto p = detail::u8(np);
  auto tv = input.native();
  b2_column* out = nullptr;
  detail::check(b2_sorted_order(&tv, o.data(), (int32_t)o.size(), p.data(), (int32_t)p.size(), stable, stream.value(), &out));
  return std::make_unique<column>(out);
}
inline std::unique_ptr<column> sorted_order(table_view const& input, CUDF_B2_SORT_ARGS) { return sorted_order_impl(input, column_order, null_precedence, false, stream); }
inline std::unique_ptr<column> stable_sorted_order(table_view const& input, CUDF_B2_SORT_ARGS) { return sorted_order_impl(input, column_order, null_precedence, true, stream); }
inline std::unique_ptr<table> sort_impl(table_view const& input, std::vector<order> const& co, std::vector<null_order> const& np,
                                        bool stable, rmm::cuda_stream_view stream)
{
  auto o = detail::u8(co); auto p = detail::u8(np);
  auto tv = input.native();
  b2_table* out = nullptr;
  detail::check(b2_sort(&tv, o.data(), (int32_t)o.size(), p.data(), (int32_t)p.size(), stable, stream.value(), &out));
  return table::from_handle(out);
}
inline std::unique_ptr<table> sort(table_view const& input, CUDF_B2_SORT_ARGS) { return sort_impl(input, column_order, null_precedence, false, stream); }
inline std::unique_ptr<table> stable_sort(table_view const& input, CUDF_B2_SORT_ARGS) { return sort_impl(input, column_order, null_precedence, true, stream); }
inline std::unique_ptr<table> sort_by_key_impl(table_view const& values, table_view const& keys, std::vector<order> const& co,
                                               std::vector<null_order> const& np, bool stable, rmm::cuda_stream_view stream)
{
  auto o = detail::u8(co); auto p = detail::u8(np);
  auto vv = values.native(); auto kv = keys.native();
  b2_table* out = nullptr;
  detail::check(b2_sort_by_key(&vv, &kv, o.data(), (int32_t)o.size(), p.data(), (int32_t)p.size(), stable, stream.value(), &out));
  return table::from_handle(out);
}
inline std::unique_ptr<table> sort_by_key(table_view const& values, table_view const& keys, CUDF_B2_SORT_ARGS) { return sort_by_key_impl(values, keys, column_order, null_precedence, false, stream); }
inline std::unique_ptr<table> stable_sort_by_key(table_view const& values, table_view const& keys, CUDF_B2_SORT_ARGS) { return sort_by_key_impl(values, keys, column_order, null_precedence, true, stream); }
// segmented sort (sorting.hpp:232-366)
inline std::unique_ptr<column> segmented_sorted_order_impl(table_view const& keys, column_view const& segment_offsets,
                                                           std::vector<order> const& co, std::vector<null_order> const& np, bool stable,
                                                           rmm::cuda_stream_view stream)
{
  auto o = detail::u8(co); auto p = detail::u8(np);
  auto kv = keys.native();
  b2_column* out = nullptr;
  detail::check(b2_segmented_sorted_order(&kv, &segment_offsets.native(), o.data(), (int32_t)o.size(), p.data(), (int32_t)p.size(), stable,
                                          stream.value(), &out));
  return std::make_unique<column>(out);
}
inline std::unique_ptr<column> segmented_sorted_order(table_view const& keys, column_view const& segment_offsets, CUDF_B2_SORT_ARGS) { return segmented_sorted_order_impl(keys, segment_offsets, column_order, null_precedence, false, stream); }
inline std::unique_ptr<column> stable_segmented_sorted_order(table_view const& keys, column_view const& segment_offsets, CUDF_B2_SORT_ARGS) { return segmented_sorted_order_impl(keys, segment_offsets, column_order, null_precedence, true, stream); }
inline std::unique_ptr<table> segmented_sort_by_key_impl(table_view const& values, table_view const& keys, column_view const& segment_offsets,
                                                         std::vector<order> const& co, std::vector<null_order> const& np, bool stable,
                                                         rmm::cuda_stream_view stream)
{
  auto o = detail::u8(co); auto p = detail::u8(np);
  auto vv = values.native(); auto kv = keys.native();
  b2_table* out = nullptr;
  detail::check(b2_segmented_sort_by_key(&vv, &kv, &segment_offsets.native(), o.data(), (int32_t)o.size(), p.data(), (int32_t)p.size(),
                                         stable, stream.value(), &out));
  return table::from_handle(out);
}
inline std::unique_ptr<table> segmented_sort_by_key(table_view const& values, table_view const& keys, column_view const& segment_offsets, CUDF_B2_SORT_ARGS) { return segmented_sort_by_key_impl(values, keys, segment_offsets, column_order, null_precedence, false, stream); }
inline std::unique_ptr<table> stable_segmented_sort_by_key(table_view const& values, table_view const& keys, column_view const& segment_offsets, CUDF_B2_SORT_ARGS) { return segmented_sort_by_key_impl(values, keys, segment_offsets, column_order, null_precedence, true, stream); }
#undef CUDF_B2_SORT_ARGS
// rank (sorting.hpp:165-230; rank_method: aggregation.hpp:37-43)
enum class rank_method : int32_t { FIRST, AVERAGE, MIN, MAX, DENSE };
inline std::unique_ptr<column> rank(column_view const& input, rank_method method, order column_order, null_policy null_handling,
                                    null_order null_precedence, bool percentage, rmm::cuda_stream_view stream = cudf::get_default_stream(),
                                    rmm::device_async_resource_ref = cudf::get_current_device_resource_ref())
{
  b2_column* out = nullptr;
  detail::check(b2_rank(&input.native(), static_cast<int32_t>(method), static_cast<int32_t>(column_order), static_cast<int32_t>(null_handling),
                        static_cast<int32_t>(null_precedence), percentage ? 1 : 0, stream.value(), &out));
  return std::make_unique<column>(out);
}
// top-k (sorting.hpp:370-416)
inline std::unique_ptr<column> top_k(column_view const& col, size_type k, order topk_order = order::DESCENDING,
                                     rmm::cuda_stream_view stream = cudf::get_default_stream(),
                                     rmm::device_async_resource_ref = cudf::get_current_device_resource_ref())
{
  b2_column* out = nullptr;
  detail::check(b2_top_k(&col.native(), k, static_cast<int32_t>(topk_order), stream.value(), &out));
  return std::make_unique<column>(out);
}
inline std::unique_ptr<column> top_k_order(column_view const& col, size_type k, order topk_order = order::DESCENDING,
                                           rmm::cuda_stream_view stream = cudf::get_default_stream(),
                                           rmm::device_async_resource_ref = cudf::get_current_device_resource_ref())
{
  b2_column* out = nullptr;
  detail::check(b2_top_k_order(&col.native(), k, static_cast<int32_t>(topk_order), stream.value(), &out));
  return std::make_unique<column>(out);
}

inline std::unique_ptr<table> gather(table_view const& source_table, column_view const& gather_map,
                                     out_of_bounds_policy bounds_policy = out_of_bounds_policy::DONT_CHECK,
                                     rmm::cuda_stream_view stream = cudf::get_default_stream(),
                                     rmm::device_async_resource_ref = cudf::get_current_device_resource_ref())
{
  auto tv = source_table.native();
  b2_table* out = nullptr;
  detail::check(b2_gather(&tv, &gather_map.native(), static_cast<int32_t>(bounds_policy), stream.value(), &out));
  return table::from_handle(out);
}

// ------------------------------------------------------------------------------------------------
// join/join.hpp, join/hash_join.hpp
// ------------------------------------------------------------------------------------------------
using join_result = std::pair<std::unique_ptr<rmm::device_uvector<size_type>>, std::unique_ptr<rmm::device_uvector<size_type>>>;
namespace detail {
inline std::unique_ptr<rmm::device_uvector<size_type>> to_uvector(b2_column* c)
{
  b2_column_view v{};
  check(b2_column_view_of(c, &v));
  return std::make_unique<rmm::device_uvector<size_type>>(c, static_cast<size_type*>(const_cast<void*>(v.data)), (std::size_t)v.size);
}
}  // namespace detail
#define CUDF_B2_FREE_JOIN(NAME)                                                                                    \
  inline join_result NAME(table_view const& left_keys, table_view const& right_keys,                               \
                          null_equality compare_nulls = null_equality::EQUAL,                                      \
                          rmm::cuda_stream_view stream = cudf::get_default_stream(),                               \
                          rmm::device_async_resource_ref = cudf::get_current_device_resource_ref())                \
  {                                                                                                                \
    auto l = left_keys.native(); auto r = right_keys.native();                                                     \
    b2_column *lo = nullptr, *ro = nullptr;                                                                        \
    detail::check(b2_##NAME(&l, &r, static_cast<int32_t>(compare_nulls), stream.value(), &lo, &ro));               \
    return {detail::to_uvector(lo), detail::to_uvector(ro)};                                                       \
  }
CUDF_B2_FREE_JOIN(inner_join)
CUDF_B2_FREE_JOIN(left_join)
CUDF_B2_FREE_JOIN(full_join)
#undef CUDF_B2_FREE_JOIN

// join.hpp:81-125
struct join_match_context {
  table_view _left_table;
  std::unique_ptr<rmm::device_uvector<size_type>> _match_counts;
  join_match_context(table_view const& left_table, std::unique_ptr<rmm::device_uvector<size_type>> match_counts)
    : _left_table{left_table}, _match_counts{std::move(match_counts)}
  {
  }
  join_match_context(join_match_context const&)            = delete;
  join_match_context& operator=(join_match_context const&) = delete;
  join_match_context(join_match_context&&)                 = default;
  join_match_context& operator=(join_match_context&&)      = default;
  virtual ~join_match_context()                            = default;
};
struct join_partition_context {
  std::unique_ptr<join_match_context> left_table_context;
  size_type left_start_idx;
  size_type left_end_idx;
};
template <typename T>
struct device_span {  // cudf::device_span<T const> over device memory owned elsewhere
  T* ptr{nullptr};
  std::size_t n{0};
  device_span() = default;
  device_span(T* p, std::size_t size) : ptr(p), n(size) {}
  template <typename U>
  device_span(rmm::device_uvector<U> const& v) : ptr(v.data()), n(v.size()) {}  // NOLINT
  [[nodiscard]] T* data() const noexcept { return ptr; }
  [[nodiscard]] std::size_t size() const noexcept { return n; }
};

class hash_join {
 public:
  hash_join() = delete;
  hash_join(hash_join const&) = delete;
  hash_join(table_view const& build, null_equality compare_nulls, rmm::cuda_stream_view stream = cudf::get_default_stream())
  {
    auto b = build.native();
    detail::check(b2_hash_join_create(&b, -1, static_cast<int32_t>(compare_nulls), 0.5, stream.value(), &h_));
  }
  hash_join(table_view const& build, nullable_join has_nulls, null_equality compare_nulls, double load_factor = 0.5,
            rmm::cuda_stream_view stream = cudf::get_default_stream())
  {
    auto b = build.native();
    detail::check(b2_hash_join_create(&b, has_nulls == nullable_join::YES ? 1 : 0, static_cast<int32_t>(compare_nulls), load_factor,
                                      stream.value(), &h_));
  }
  ~hash_join() { if (h_) b2_hash_join_destroy(h_); }
#define CUDF_B2_OBJ_JOIN(NAME)                                                                                       \
  [[nodiscard]] join_result NAME(table_view const& probe, std::optional<std::size_t> output_size = {},               \
                                 rmm::cuda_stream_view stream = cudf::get_default_stream(),                          \
                                 rmm::device_async_resource_ref = cudf::get_current_device_resource_ref()) const     \
  {                                                                                                                  \
    auto p = probe.native();                                                                                         \
    b2_column *lo = nullptr, *ro = nullptr;                                                                          \
    detail::check(b2_hash_join_##NAME(h_, &p, output_size.has_value(), output_size.value_or(0), stream.value(), &lo, &ro)); \
    return {detail::to_uvector(lo), detail::to_uvector(ro)};                                                         \
  }                                                                                                                  \
  [[nodiscard]] std::size_t NAME##_size(table_view const& probe, rmm::cuda_stream_view stream = cudf::get_default_stream()) const \
  {                                                                                                                  \
    auto p = probe.native();                                                                                         \
    std::size_t out = 0;                                                                                             \
    detail::check(b2_hash_join_##NAME##_size(h_, &p, stream.value(), &out));                                         \
    return out;                                                                                                      \
  }
  CUDF_B2_OBJ_JOIN(inner_join)
  CUDF_B2_OBJ_JOIN(left_join)
  CUDF_B2_OBJ_JOIN(full_join)
#undef CUDF_B2_OBJ_JOIN
  // match context + partitioned probes (hash_join.hpp:254-440)
#define CUDF_B2_MATCH_CTX(NAME, KIND)                                                                                \
  [[nodiscard]] cudf::join_match_context NAME##_match_context(table_view const& left,                                \
                                                              rmm::cuda_stream_view stream = cudf::get_default_stream(), \
                                                              rmm::device_async_resource_ref = cudf::get_current_device_resource_ref()) const \
  {                                                                                                                  \
    auto p = left.native();                                                                                          \
    b2_column* c = nullptr;                                                                                          \
    detail::check(b2_hash_join_match_counts(h_, &p, KIND, stream.value(), &c));                                      \
    return cudf::join_match_context{left, detail::to_uvector(c)};                                                    \
  }                                                                                                                  \
  [[nodiscard]] join_result partitioned_##NAME(cudf::join_partition_context const& context,                          \
                                               rmm::cuda_stream_view stream = cudf::get_default_stream(),            \
                                               rmm::device_async_resource_ref = cudf::get_current_device_resource_ref()) const \
  {                                                                                                                  \
    if (!context.left_table_context || !context.left_table_context->_match_counts)                                   \
      throw std::invalid_argument("join_partition_context without a match context");                                 \
    auto const& ctx = *context.left_table_context;                                                                   \
    auto p = ctx._left_table.native();                                                                               \
    b2_column_view counts{B2_INT32, (int32_t)ctx._match_counts->size(), ctx._match_counts->data(), nullptr, 0, 0};   \
    b2_column *lo = nullptr, *ro = nullptr;                                                                          \
    detail::check(b2_hash_join_partitioned_join(h_, &p, &counts, context.left_start_idx, context.left_end_idx, KIND, \
                                                stream.value(), &lo, &ro));                                          \
    return {detail::to_uvector(lo), detail::to_uvector(ro)};                                                         \
  }
  CUDF_B2_MATCH_CTX(inner_join, 0)
  CUDF_B2_MATCH_CTX(left_join, 1)
  CUDF_B2_MATCH_CTX(full_join, 2)
#undef CUDF_B2_MATCH_CTX
  [[nodiscard]] static join_result finalize_partitioned_full_join(std::vector<device_span<size_type const>> const& left_partials,
                                                                  std::vector<device_span<size_type const>> const& right_partials,
                                                                  size_type left_table_num_rows, size_type right_table_num_rows,
                                                                  rmm::cuda_stream_view stream = cudf::get_default_stream(),
                                                                  rmm::device_async_resource_ref = cudf::get_current_device_resource_ref())
  {
    if (left_partials.size() != right_partials.size()) throw std::invalid_argument("left and right partials differ in number");
    std::vector<b2_column_view> l, r;
    for (std::size_t i = 0; i < left_partials.size(); ++i) {
      l.push_back(b2_column_view{B2_INT32, (int32_t)left_partials[i].size(), left_partials[i].data(), nullptr, 0, 0});
      r.push_back(b2_column_view{B2_INT32, (int32_t)right_partials[i].size(), right_partials[i].data(), nullptr, 0, 0});
    }
    b2_column *lo = nullptr, *ro = nullptr;
    detail::check(b2_hash_join_finalize_full_join(l.data(), r.data(), (int32_t)l.size(), left_table_num_rows, right_table_num_rows,
                                                  stream.value(), &lo, &ro));
    return {detail::to_uvector(lo), detail::to_uvector(ro)};
  }

 private:
  b2_hash_join* h_{nullptr};
};

// join/filtered_join.hpp: left semi / anti join against a right (filter) table built once; results are the left row
// indices in ascending order. load_factor outside (0, 1] is std::invalid_argument.
class filtered_join {
 public:
  filtered_join() = delete;
  filtered_join(filtered_join const&)            = delete;
  filtered_join(filtered_join&&)                 = delete;
  filtered_join& operator=(filtered_join const&) = delete;
  filtered_join& operator=(filtered_join&&)      = delete;
  filtered_join(table_view const& right, null_equality compare_nulls, rmm::cuda_stream_view stream)
    : filtered_join(right, compare_nulls, 0.5, stream)
  {
  }
  filtered_join(table_view const& right, null_equality compare_nulls, double load_factor, rmm::cuda_stream_view stream)
  {
    auto r = right.native();
    detail::check(b2_filtered_join_create(&r, static_cast<int32_t>(compare_nulls), load_factor, stream.value(), &h_));
  }
  ~filtered_join() { if (h_) b2_filtered_join_destroy(h_); }
  [[nodiscard]] std::unique_ptr<rmm::device_uvector<size_type>> semi_join(
    table_view const& left, rmm::cuda_stream_view stream = cudf::get_default_stream(),
    rmm::device_async_resource_ref = cudf::get_current_device_resource_ref()) const
  {
    auto l = left.native();
    b2_column* out = nullptr;
    detail::check(b2_filtered_join_semi_join(h_, &l, stream.value(), &out));
    return detail::to_uvector(out);
  }
  [[nodiscard]] std::unique_ptr<rmm::device_uvector<size_type>> anti_join(
    table_view const& left, rmm::cuda_stream_view stream = cudf::get_default_stream(),
    rmm::device_async_resource_ref = cudf::get_current_device_resource_ref()) const
  {
    auto l = left.native();
    b2_column* out = nullptr;
    detail::check(b2_filtered_join_anti_join(h_, &l, stream.value(), &out));
    return detail::to_uvector(out);
  }

 private:
  b2_filtered_join* h_{nullptr};
};

// ------------------------------------------------------------------------------------------------
// groupby.hpp
// ------------------------------------------------------------------------------------------------
namespace groupby {
struct aggregation_request {
  column_view values;
  std::vector<std::unique_ptr<groupby_aggregation>> aggregations;
};
struct scan_request {
  column_view values;
  std::vector<std::unique_ptr<groupby_scan_aggregation>> aggregations;
};
struct aggregation_result {
  std::vector<std::unique_ptr<column>> results{};
};
class groupby {
 public:
  groupby() = delete;
  groupby(groupby const&) = delete;
  explicit groupby(table_view const& keys, null_policy null_handling = null_policy::EXCLUDE, sorted keys_are_sorted = sorted::NO,
                   std::vector<order> const& column_order = {}, std::vector<null_order> const& null_precedence = {})
    : keys_(keys)
  {
    auto o = cudf::detail::u8(column_order); auto p = cudf::detail::u8(null_precedence);
    auto k = keys_.native();
    cudf::detail::check(b2_groupby_create(&k, static_cast<int32_t>(null_handling), static_cast<int32_t>(keys_are_sorted), o.data(),
                                          (int32_t)o.size(), p.data(), (int32_t)p.size(), &h_));
  }
  ~groupby() { if (h_) b2_groupby_destroy(h_); }

  template <typename Request>
  std::pair<std::unique_ptr<table>, std::vector<aggregation_result>> run(std::vector<Request> const& requests, bool is_scan,
                                                                         rmm::cuda_stream_view stream)
  {
    std::vector<std::vector<int32_t>> kinds(requests.size());
    std::vector<b2_agg_request> raw;
    for (std::size_t i = 0; i < requests.size(); ++i) {
      for (auto const& a : requests[i].aggregations) kinds[i].push_back(a->abi_kind());
      raw.push_back(b2_agg_request{requests[i].values.native(), kinds[i].data(), (int32_t)kinds[i].size()});
    }
    b2_table *ko = nullptr, *ro = nullptr;
    cudf::detail::check((is_scan ? b2_groupby_scan : b2_groupby_aggregate)(h_, raw.data(), (int32_t)raw.size(), stream.value(), &ko, &ro));
    auto flat = table::from_handle(ro)->release();
    std::vector<aggregation_result> results(requests.size());
    std::size_t k = 0;
    for (std::size_t i = 0; i < requests.size(); ++i)
      for (std::size_t j = 0; j < requests[i].aggregations.size(); ++j) results[i].results.push_back(std::move(flat[k++]));
    return {table::from_handle(ko), std::move(results)};
  }
  std::pair<std::unique_ptr<table>, std::vector<aggregation_result>> aggregate(
    std::vector<aggregation_request> const& requests, rmm::cuda_stream_view stream = cudf::get_default_stream(),
    rmm::device_async_resource_ref = cudf::get_current_device_resource_ref())
  {
    return run(requests, false, stream);
  }
  std::pair<std::unique_ptr<table>, std::vector<aggregation_result>> scan(
    std::vector<scan_request> const& requests, rmm::cuda_stream_view stream = cudf::get_default_stream(),
    rmm::device_async_resource_ref = cudf::get_current_device_resource_ref())
  {
    return run(requests, true, stream);
  }
 private:
  table_view keys_;
  b2_groupby* h_{nullptr};
};
}  // namespace groupby

// ------------------------------------------------------------------------------------------------
// reduction.hpp
// ------------------------------------------------------------------------------------------------
inline std::unique_ptr<scalar> reduce(column_view const& col, reduce_aggregation const& agg, data_type output_dtype,
                                      std::optional<std::reference_wrapper<scalar const>> init,
                                      rmm::cuda_stream_view stream = cudf::get_default_stream(),
                                      rmm::device_async_resource_ref = cudf::get_current_device_resource_ref())
{
  b2_scalar* out = nullptr;
  detail::check(b2_reduce(&col.native(), static_cast<int32_t>(agg.kind), static_cast<int32_t>(output_dtype.id()),
                          init.has_value() ? init->get().native() : nullptr, stream.value(), &out));
  return std::make_unique<scalar>(out);
}
inline std::unique_ptr<scalar> reduce(column_view const& col, reduce_aggregation const& agg, data_type output_dtype,
                                      rmm::cuda_stream_view stream = cudf::get_default_stream(),
                                      rmm::device_async_resource_ref mr = cudf::get_current_device_resource_ref())
{
  return reduce(col, agg, output_dtype, std::nullopt, stream, mr);
}
inline std::unique_ptr<column> scan(column_view const& input, scan_aggregation const& agg, scan_type inclusive,
                                    null_policy null_handling = null_policy::EXCLUDE,
                                    rmm::cuda_stream_view stream = cudf::get_default_stream(),
                                    rmm::device_async_resource_ref = cudf::get_current_device_resource_ref())
{
  b2_column* out = nullptr;
  detail::check(b2_scan(&input.native(), static_cast<int32_t>(agg.kind), static_cast<int32_t>(inclusive),
                        static_cast<int32_t>(null_handling), stream.value(), &out));
  return std::make_unique<column>(out);
}
struct device_span_size_type { size_type const* ptr; std::size_t n; };  // cudf::device_span<size_type const>
inline std::unique_ptr<column> segmented_reduce(column_view const& segmented_values, device_span_size_type offsets,
                                                segmented_reduce_aggregation const& agg, data_type output_dtype,
                                                null_policy null_handling,
                                                std::optional<std::reference_wrapper<scalar const>> init = std::nullopt,
                                                rmm::cuda_stream_view stream = cudf::get_default_stream(),
                                                rmm::device_async_resource_ref = cudf::get_current_device_resource_ref())
{
  b2_column* out = nullptr;
  detail::check(b2_segmented_reduce(&segmented_values.native(), offsets.ptr, (int32_t)offsets.n, static_cast<int32_t>(agg.kind),
                                    static_cast<int32_t>(output_dtype.id()), static_cast<int32_t>(null_handling),
                                    init.has_value() ? init->get().native() : nullptr, stream.value(), &out));
  return std::make_unique<column>(out);
}

// ------------------------------------------------------------------------------------------------
// null_mask.hpp
// ------------------------------------------------------------------------------------------------
inline std::size_t bitmask_allocation_size_bytes(size_type number_of_bits) { return b2_bitmask_allocation_size_bytes(number_of_bits); }
inline rmm::device_buffer create_null_mask(size_type size, mask_state state, rmm::cuda_stream_view stream = cudf::get_default_stream())
{
  b2_buffer* out = nullptr;
  detail::check(b2_create_null_mask(size, static_cast<int32_t>(state), stream.value(), &out));
  return rmm::device_buffer{out};
}
inline void set_null_mask(bitmask_type* bitmask, size_type begin_bit, size_type end_bit, bool valid,
                          rmm::cuda_stream_view stream = cudf::get_default_stream())
{
  detail::check(b2_set_null_mask(bitmask, begin_bit, end_bit, valid, stream.value()));
}
inline rmm::device_buffer copy_bitmask(column_view const& view, rmm::cuda_stream_view stream = cudf::get_default_stream())
{
  b2_buffer* out = nullptr;
  detail::check(b2_copy_bitmask(view.null_mask(), view.offset(), view.offset() + view.size(), stream.value(), &out));
  return rmm::device_buffer{out};
}
inline size_type null_count(bitmask_type const* bitmask, size_type start, size_type stop,
                            rmm::cuda_stream_view stream = cudf::get_default_stream())
{
  int32_t out = 0;
  detail::check(b2_null_count(bitmask, start, stop, stream.value(), &out));
  return out;
}
inline std::pair<rmm::device_buffer, size_type> bitmask_and(table_view const& view, rmm::cuda_stream_view stream = cudf::get_default_stream())
{
  auto tv = view.native();
  b2_buffer* out = nullptr;
  int32_t nulls = 0;
  detail::check(b2_bitmask_and(&tv, stream.value(), &out, &nulls));
  return {rmm::device_buffer{out}, nulls};
}


// ------------------------------------------------------------------------------------------------
// partitioning.hpp (cpp/include/cudf/partitioning.hpp:32-175)
// ------------------------------------------------------------------------------------------------
enum class hash_id : int32_t { HASH_IDENTITY = 0, HASH_MURMUR3 };
static constexpr uint32_t DEFAULT_HASH_SEED = 0;

inline std::pair<std::unique_ptr<table>, std::vector<size_type>> partition(table_view const& t, column_view const& partition_map,
                                                                           size_type num_partitions,
                                                                           rmm::cuda_stream_view stream = cudf::get_default_stream(),
                                                                           rmm::device_async_resource_ref = cudf::get_current_device_resource_ref())
{
  if (t.num_rows() != partition_map.size()) throw cudf::logic_error("Size mismatch between table and partition map.");
  auto tv = t.native();
  b2_table* out = nullptr;
  std::vector<size_type> offsets(static_cast<size_t>(std::max(num_partitions, 0)) + 1, 0);
  detail::check(b2_partition_by_map(&tv, &partition_map.native(), num_partitions, stream.value(), &out, offsets.data()));
  return {table::from_handle(out), std::move(offsets)};
}

inline std::pair<std::unique_ptr<table>, std::vector<size_type>> hash_partition(table_view const& input, table_view const& keys, int num_partitions,
                                                                                hash_id hash_function = hash_id::HASH_MURMUR3,
                                                                                uint32_t seed = DEFAULT_HASH_SEED,
                                                                                rmm::cuda_stream_view stream = cudf::get_default_stream(),
                                                                                rmm::device_async_resource_ref = cudf::get_current_device_resource_ref())
{
  auto tv = input.native();
  auto kv = keys.native();
  b2_table* out = nullptr;
  std::vector<size_type> offsets(static_cast<size_t>(std::max(num_partitions, 0)) + 1, 0);
  detail::check(b2_hash_partition(&tv, &kv, num_partitions, static_cast<int32_t>(hash_function), seed, stream.value(), &out, offsets.data()));
  return {table::from_handle(out), std::move(offsets)};
}
inline std::pair<std::unique_ptr<table>, std::vector<size_type>> hash_partition(table_view const& input, std::vector<size_type> const& columns_to_hash,
                                                                                int num_partitions, hash_id hash_function = hash_id::HASH_MURMUR3,
                                                                                uint32_t seed = DEFAULT_HASH_SEED,
                                                                                rmm::cuda_stream_view stream = cudf::get_default_stream(),
                                                                                rmm::device_async_resource_ref mr = cudf::get_current_device_resource_ref())
{
  std::vector<column_view> kc;
  for (auto i : columns_to_hash) kc.push_back(input.column(i));  // std::out_of_range on a bad index, as in libcudf
  return hash_partition(input, table_view{kc}, num_partitions, hash_function, seed, stream, mr);
}

// ------------------------------------------------------------------------------------------------
// contiguous_split.hpp: pack / unpack (cpp/include/cudf/contiguous_split.hpp:100-120,233-317)
// ------------------------------------------------------------------------------------------------
struct packed_columns {
  std::unique_ptr<std::vector<uint8_t>> metadata = std::make_unique<std::vector<uint8_t>>();
  std::unique_ptr<rmm::device_buffer> gpu_data   = std::make_unique<rmm::device_buffer>();
};
inline std::size_t packed_size(table_view const& input, rmm::cuda_stream_view = cudf::get_default_stream(),
                               rmm::device_async_resource_ref = cudf::get_current_device_resource_ref())
{
  auto tv = input.native();
  std::size_t bytes = 0;
  detail::check(b2_packed_size(&tv, &bytes));
  return bytes;
}
inline packed_columns pack(table_view const& input, rmm::cuda_stream_view stream = cudf::get_default_stream(),
                           rmm::device_async_resource_ref = cudf::get_current_device_resource_ref())
{
  auto tv = input.native();
  packed_columns out;
  out.metadata->resize(16 + 40 * static_cast<size_t>(input.num_columns()));
  std::size_t md = 0;
  b2_buffer* buf = nullptr;
  detail::check(b2_pack(&tv, stream.value(), out.metadata->data(), out.metadata->size(), &md, &buf));
  out.metadata->resize(md);
  out.gpu_data = std::make_unique<rmm::device_buffer>(buf);
  return out;
}
inline std::vector<uint8_t> pack_metadata(table_view const& table, uint8_t const* contiguous_buffer, size_t buffer_size)
{
  auto tv = table.native();
  std::vector<uint8_t> md(16 + 40 * static_cast<size_t>(table.num_columns()));
  std::size_t n = 0;
  detail::check(b2_pack_metadata(&tv, contiguous_buffer, buffer_size, md.data(), md.size(), &n));
  md.resize(n);
  return md;
}
inline table_view unpack(uint8_t const* metadata, size_t metadata_size, uint8_t const* gpu_data)
{
  std::vector<b2_column_view> raw(metadata_size >= 16 ? (metadata_size - 16) / 40 + 1 : 1);
  int32_t ncols = 0, nrows = 0;
  detail::check(b2_unpack(metadata, metadata_size, gpu_data, raw.data(), static_cast<int32_t>(raw.size()), &ncols, &nrows));
  std::vector<column_view> cols;
  for (int32_t i = 0; i < ncols; ++i)
    cols.emplace_back(data_type{static_cast<type_id>(raw[i].type_id)}, raw[i].size, raw[i].data, raw[i].null_mask, raw[i].null_count, 0);
  return table_view{cols};
}
inline table_view unpack(packed_columns const& input)
{
  return unpack(input.metadata->data(), input.metadata->size(), static_cast<uint8_t const*>(input.gpu_data->data()));
}

// ------------------------------------------------------------------------------------------------
// stream_compaction.hpp (cpp/include/cudf/stream_compaction.hpp:73-390): fixed-width columns, at most 8 key columns
// ------------------------------------------------------------------------------------------------
enum class duplicate_keep_option : int32_t { KEEP_ANY = 0, KEEP_FIRST, KEEP_LAST, KEEP_NONE };
namespace detail {
template <typename F>
inline std::unique_ptr<table> table_call(F&& f)
{
  b2_table* out = nullptr;
  check(f(&out));
  return table::from_handle(out);
}
}  // namespace detail
inline std::unique_ptr<table> drop_nulls(table_view const& input, std::vector<size_type> const& keys, size_type keep_threshold,
                                         rmm::cuda_stream_view stream = cudf::get_default_stream(),
                                         rmm::device_async_resource_ref = cudf::get_current_device_resource_ref())
{
  auto tv = input.native();
  return detail::table_call([&](b2_table** o) {
    return b2_drop_nulls(&tv, keys.data(), static_cast<int32_t>(keys.size()), keep_threshold, stream.value(), o);
  });
}
inline std::unique_ptr<table> drop_nulls(table_view const& input, std::vector<size_type> const& keys,
                                         rmm::cuda_stream_view stream = cudf::get_default_stream(),
                                         rmm::device_async_resource_ref mr = cudf::get_current_device_resource_ref())
{
  return drop_nulls(input, keys, static_cast<size_type>(keys.size()), stream, mr);
}
inline std::unique_ptr<table> drop_nans(table_view const& input, std::vector<size_type> const& keys, size_type keep_threshold,
                                        rmm::cuda_stream_view stream = cudf::get_default_stream(),
                                        rmm::device_async_resource_ref = cudf::get_current_device_resource_ref())
{
  auto tv = input.native();
  return detail::table_call([&](b2_table** o) {
    return b2_drop_nans(&tv, keys.data(), static_cast<int32_t>(keys.size()), keep_threshold, stream.value(), o);
  });
}
inline std::unique_ptr<table> drop_nans(table_view const& input, std::vector<size_type> const& keys,
                                        rmm::cuda_stream_view stream = cudf::get_default_stream(),
                                        rmm::device_async_resource_ref mr = cudf::get_current_device_resource_ref())
{
  return drop_nans(input, keys, static_cast<size_type>(keys.size()), stream, mr);
}
inline std::unique_ptr<table> apply_boolean_mask(table_view const& input, column_view const& boolean_mask,
                                                 rmm::cuda_stream_view stream = cudf::get_default_stream(),
                                                 rmm::device_async_resource_ref = cudf::get_current_device_resource_ref())
{
  auto tv = input.native();
  return detail::table_call([&](b2_table** o) { return b2_apply_boolean_mask(&tv, &boolean_mask.native(), 0, stream.value(), o); });
}
inline std::unique_ptr<table> apply_deletion_mask(table_view const& input, column_view const& deletion_mask,
                                                  rmm::cuda_stream_view stream = cudf::get_default_stream(),
                                                  rmm::device_async_resource_ref = cudf::get_current_device_resource_ref())
{
  auto tv = input.native();
  return detail::table_call([&](b2_table** o) { return b2_apply_boolean_mask(&tv, &deletion_mask.native(), 1, stream.value(), o); });
}
inline std::unique_ptr<table> unique(table_view const& input, std::vector<size_type> const& keys, duplicate_keep_option keep,
                                     null_equality nulls_equal = null_equality::EQUAL,
                                     rmm::cuda_stream_view stream = cudf::get_default_stream(),
                                     rmm::device_async_resource_ref = cudf::get_current_device_resource_ref())
{
  auto tv = input.native();
  return detail::table_call([&](b2_table** o) {
    return b2_unique(&tv, keys.data(), static_cast<int32_t>(keys.size()), static_cast<int32_t>(keep), static_cast<int32_t>(nulls_equal),
                     stream.value(), o);
  });
}
#define CUDF_B2_DISTINCT(NAME, STABLE)                                                                                              \
  inline std::unique_ptr<table> NAME(table_view const& input, std::vector<size_type> const& keys,                                   \
                                     duplicate_keep_option keep = duplicate_keep_option::KEEP_ANY,                                  \
                                     null_equality nulls_equal = null_equality::EQUAL, nan_equality nans_equal = nan_equality::ALL_EQUAL, \
                                     rmm::cuda_stream_view stream = cudf::get_default_stream(),                                     \
                                     rmm::device_async_resource_ref = cudf::get_current_device_resource_ref())                      \
  {                                                                                                                                 \
    auto tv = input.native();                                                                                                       \
    return detail::table_call([&](b2_table** o) {                                                                                   \
      return b2_distinct(&tv, keys.data(), static_cast<int32_t>(keys.size()), static_cast<int32_t>(keep),                           \
                         static_cast<int32_t>(nulls_equal), static_cast<int32_t>(nans_equal), STABLE, stream.value(), o);           \
    });                                                                                                                             \
  }
CUDF_B2_DISTINCT(distinct, 0)
CUDF_B2_DISTINCT(stable_distinct, 1)
#undef CUDF_B2_DISTINCT
inline std::unique_ptr<column> distinct_indices(table_view const& input, duplicate_keep_option keep = duplicate_keep_option::KEEP_ANY,
                                                null_equality nulls_equal = null_equality::EQUAL,
                                                nan_equality nans_equal = nan_equality::ALL_EQUAL,
                                                rmm::cuda_stream_view stream = cudf::get_default_stream(),
                                                rmm::device_async_resource_ref = cudf::get_current_device_resource_ref())
{
  auto tv = input.native();
  b2_column* out = nullptr;
  detail::check(b2_distinct_indices(&tv, static_cast<int32_t>(keep), static_cast<int32_t>(nulls_equal), static_cast<int32_t>(nans_equal),
                                    stream.value(), &out));
  return std::make_unique<column>(out);
}

// binaryop.hpp (cpp/include/cudf/binaryop.hpp:30-84,158-294): fixed-width columns and scalars; the semantics, undefined values
// and errors are b2_binary_operation's (include/cudf_b200.h). An unsupported combination is cudf::data_type_error, differing
// column sizes std::invalid_argument, a type id outside type_id cudf::logic_error.
enum class binary_operator : int32_t {
  ADD, SUB, MUL, DIV, TRUE_DIV, FLOOR_DIV, MOD, PMOD, PYMOD, POW, INT_POW, LOG_BASE, ATAN2, SHIFT_LEFT, SHIFT_RIGHT,
  SHIFT_RIGHT_UNSIGNED, BITWISE_AND, BITWISE_OR, BITWISE_XOR, LOGICAL_AND, LOGICAL_OR, EQUAL, NOT_EQUAL, LESS, GREATER,
  LESS_EQUAL, GREATER_EQUAL, NULL_EQUALS, NULL_NOT_EQUALS, NULL_MAX, NULL_MIN, GENERIC_BINARY, NULL_LOGICAL_AND,
  NULL_LOGICAL_OR, INVALID_BINARY
};
inline std::unique_ptr<column> binary_operation(scalar const& lhs, column_view const& rhs, binary_operator op, data_type output_type,
                                                rmm::cuda_stream_view stream = cudf::get_default_stream(),
                                                rmm::device_async_resource_ref = cudf::get_current_device_resource_ref())
{
  b2_column* out = nullptr;
  detail::check(b2_binary_operation_sc(lhs.native(), &rhs.native(), static_cast<int32_t>(op), static_cast<int32_t>(output_type.id()),
                                       stream.value(), &out));
  return std::make_unique<column>(out);
}
inline std::unique_ptr<column> binary_operation(column_view const& lhs, scalar const& rhs, binary_operator op, data_type output_type,
                                                rmm::cuda_stream_view stream = cudf::get_default_stream(),
                                                rmm::device_async_resource_ref = cudf::get_current_device_resource_ref())
{
  b2_column* out = nullptr;
  detail::check(b2_binary_operation_cs(&lhs.native(), rhs.native(), static_cast<int32_t>(op), static_cast<int32_t>(output_type.id()),
                                       stream.value(), &out));
  return std::make_unique<column>(out);
}
inline std::unique_ptr<column> binary_operation(column_view const& lhs, column_view const& rhs, binary_operator op,
                                                data_type output_type, rmm::cuda_stream_view stream = cudf::get_default_stream(),
                                                rmm::device_async_resource_ref = cudf::get_current_device_resource_ref())
{
  b2_column* out = nullptr;
  detail::check(b2_binary_operation(&lhs.native(), &rhs.native(), static_cast<int32_t>(op), static_cast<int32_t>(output_type.id()),
                                    stream.value(), &out));
  return std::make_unique<column>(out);
}
namespace binops {
inline bool is_supported_operation(data_type out, data_type lhs, data_type rhs, binary_operator op)
{
  int32_t r = 0;
  detail::check(b2_binary_is_supported_operation(static_cast<int32_t>(out.id()), static_cast<int32_t>(lhs.id()),
                                                 static_cast<int32_t>(rhs.id()), static_cast<int32_t>(op), &r));
  return r != 0;
}
}  // namespace binops

// unary.hpp (cpp/include/cudf/unary.hpp:32-57,60-164): fixed-width columns; the semantics, undefined values and errors are
// b2_unary_operation's and b2_cast's (include/cudf_b200.h).  An unsupported (op, type) pair, an op outside the enum, a
// timestamp <-> numeric cast and a non-fixed-width cast target are cudf::logic_error; decimal, dictionary, string and nested
// types cudf::data_type_error.  Deviation: is_supported_cast is false for decimal types (the reference casts them).
enum class unary_operator : int32_t {
  SIN, COS, TAN, ARCSIN, ARCCOS, ARCTAN, SINH, COSH, TANH, ARCSINH, ARCCOSH, ARCTANH, EXP, LOG, SQRT, CBRT, CEIL, FLOOR, ABS,
  RINT, BIT_COUNT, BIT_INVERT, NOT, NEGATE
};
inline std::unique_ptr<column> unary_operation(column_view const& input, unary_operator op,
                                               rmm::cuda_stream_view stream = cudf::get_default_stream(),
                                               rmm::device_async_resource_ref = cudf::get_current_device_resource_ref())
{
  b2_column* out = nullptr;
  detail::check(b2_unary_operation(&input.native(), static_cast<int32_t>(op), stream.value(), &out));
  return std::make_unique<column>(out);
}
inline std::unique_ptr<column> is_null(column_view const& input, rmm::cuda_stream_view stream = cudf::get_default_stream(),
                                       rmm::device_async_resource_ref = cudf::get_current_device_resource_ref())
{
  b2_column* out = nullptr;
  detail::check(b2_is_null(&input.native(), stream.value(), &out));
  return std::make_unique<column>(out);
}
inline std::unique_ptr<column> is_valid(column_view const& input, rmm::cuda_stream_view stream = cudf::get_default_stream(),
                                        rmm::device_async_resource_ref = cudf::get_current_device_resource_ref())
{
  b2_column* out = nullptr;
  detail::check(b2_is_valid(&input.native(), stream.value(), &out));
  return std::make_unique<column>(out);
}
inline std::unique_ptr<column> cast(column_view const& input, data_type out_type,
                                    rmm::cuda_stream_view stream = cudf::get_default_stream(),
                                    rmm::device_async_resource_ref = cudf::get_current_device_resource_ref())
{
  b2_column* out = nullptr;
  detail::check(b2_cast(&input.native(), static_cast<int32_t>(out_type.id()), stream.value(), &out));
  return std::make_unique<column>(out);
}
inline bool is_supported_cast(data_type from, data_type to) noexcept
{
  int32_t r = 0;
  return b2_is_supported_cast(static_cast<int32_t>(from.id()), static_cast<int32_t>(to.id()), &r) == B2_OK && r != 0;
}
inline std::unique_ptr<column> is_nan(column_view const& input, rmm::cuda_stream_view stream = cudf::get_default_stream(),
                                      rmm::device_async_resource_ref = cudf::get_current_device_resource_ref())
{
  b2_column* out = nullptr;
  detail::check(b2_is_nan(&input.native(), stream.value(), &out));
  return std::make_unique<column>(out);
}
inline std::unique_ptr<column> is_not_nan(column_view const& input, rmm::cuda_stream_view stream = cudf::get_default_stream(),
                                          rmm::device_async_resource_ref = cudf::get_current_device_resource_ref())
{
  b2_column* out = nullptr;
  detail::check(b2_is_not_nan(&input.native(), stream.value(), &out));
  return std::make_unique<column>(out);
}

// utilities/traits.hpp:681 and column/column_view.hpp:714-759: both types fixed-width with the same storage width (decimal
// types are not held here, so none is bit-castable); bit_cast is a zero-copy view of the same data and mask
namespace detail {
constexpr int fixed_width_bytes(type_id t)
{
  switch (t) {
    case type_id::INT8: case type_id::UINT8: case type_id::BOOL8: return 1;
    case type_id::INT16: case type_id::UINT16: return 2;
    case type_id::INT32: case type_id::UINT32: case type_id::FLOAT32: case type_id::TIMESTAMP_DAYS: case type_id::DURATION_DAYS:
      return 4;
    case type_id::INT64: case type_id::UINT64: case type_id::FLOAT64: case type_id::TIMESTAMP_SECONDS:
    case type_id::TIMESTAMP_MILLISECONDS: case type_id::TIMESTAMP_MICROSECONDS: case type_id::TIMESTAMP_NANOSECONDS:
    case type_id::DURATION_SECONDS: case type_id::DURATION_MILLISECONDS: case type_id::DURATION_MICROSECONDS:
    case type_id::DURATION_NANOSECONDS: return 8;
    default: return 0;
  }
}
}  // namespace detail
inline bool is_bit_castable(data_type from, data_type to)
{
  int const w = detail::fixed_width_bytes(from.id());
  return w != 0 && w == detail::fixed_width_bytes(to.id());
}
inline column_view bit_cast(column_view const& input, data_type type)
{
  if (!is_bit_castable(input.type(), type)) throw cudf::logic_error("types are not bit-castable");
  return column_view{type, input.size(), input.head<void>(), input.null_mask(), input.null_count(), input.offset()};
}

// replace.hpp (cpp/include/cudf/replace.hpp): fixed-width columns; the semantics and errors are b2_replace_nulls*',
// b2_replace_nans*', b2_find_and_replace_all's, b2_clamp's and b2_normalize_nans_and_zeros*' (include/cudf_b200.h).  LOGIC is
// cudf::logic_error and DATA_TYPE cudf::data_type_error.
enum class replace_policy : bool { PRECEDING, FOLLOWING };
inline std::unique_ptr<column> replace_nulls(column_view const& input, column_view const& replacement,
                                             rmm::cuda_stream_view stream = cudf::get_default_stream(),
                                             rmm::device_async_resource_ref = cudf::get_current_device_resource_ref())
{
  b2_column* out = nullptr;
  detail::check(b2_replace_nulls(&input.native(), &replacement.native(), stream.value(), &out));
  return std::make_unique<column>(out);
}
inline std::unique_ptr<column> replace_nulls(column_view const& input, scalar const& replacement,
                                             rmm::cuda_stream_view stream = cudf::get_default_stream(),
                                             rmm::device_async_resource_ref = cudf::get_current_device_resource_ref())
{
  b2_column* out = nullptr;
  detail::check(b2_replace_nulls_scalar(&input.native(), replacement.native(), stream.value(), &out));
  return std::make_unique<column>(out);
}
inline std::unique_ptr<column> replace_nulls(column_view const& input, replace_policy const& policy,
                                             rmm::cuda_stream_view stream = cudf::get_default_stream(),
                                             rmm::device_async_resource_ref = cudf::get_current_device_resource_ref())
{
  b2_column* out = nullptr;
  detail::check(b2_replace_nulls_policy(&input.native(), policy == replace_policy::PRECEDING ? B2_REPLACE_PRECEDING : B2_REPLACE_FOLLOWING,
                                        stream.value(), &out));
  return std::make_unique<column>(out);
}
inline std::unique_ptr<column> replace_nans(column_view const& input, column_view const& replacement,
                                            rmm::cuda_stream_view stream = cudf::get_default_stream(),
                                            rmm::device_async_resource_ref = cudf::get_current_device_resource_ref())
{
  b2_column* out = nullptr;
  detail::check(b2_replace_nans(&input.native(), &replacement.native(), stream.value(), &out));
  return std::make_unique<column>(out);
}
inline std::unique_ptr<column> replace_nans(column_view const& input, scalar const& replacement,
                                            rmm::cuda_stream_view stream = cudf::get_default_stream(),
                                            rmm::device_async_resource_ref = cudf::get_current_device_resource_ref())
{
  b2_column* out = nullptr;
  detail::check(b2_replace_nans_scalar(&input.native(), replacement.native(), stream.value(), &out));
  return std::make_unique<column>(out);
}
inline std::unique_ptr<column> find_and_replace_all(column_view const& input_col, column_view const& values_to_replace,
                                                    column_view const& replacement_values,
                                                    rmm::cuda_stream_view stream = cudf::get_default_stream(),
                                                    rmm::device_async_resource_ref = cudf::get_current_device_resource_ref())
{
  b2_column* out = nullptr;
  detail::check(b2_find_and_replace_all(&input_col.native(), &values_to_replace.native(), &replacement_values.native(), stream.value(),
                                        &out));
  return std::make_unique<column>(out);
}
inline std::unique_ptr<column> clamp(column_view const& input, scalar const& lo, scalar const& lo_replace, scalar const& hi,
                                     scalar const& hi_replace, rmm::cuda_stream_view stream = cudf::get_default_stream(),
                                     rmm::device_async_resource_ref = cudf::get_current_device_resource_ref())
{
  b2_column* out = nullptr;
  detail::check(b2_clamp(&input.native(), lo.native(), lo_replace.native(), hi.native(), hi_replace.native(), stream.value(), &out));
  return std::make_unique<column>(out);
}
inline std::unique_ptr<column> clamp(column_view const& input, scalar const& lo, scalar const& hi,
                                     rmm::cuda_stream_view stream = cudf::get_default_stream(),
                                     rmm::device_async_resource_ref mr = cudf::get_current_device_resource_ref())
{
  return clamp(input, lo, lo, hi, hi, stream, mr);
}
inline std::unique_ptr<column> normalize_nans_and_zeros(column_view const& input,
                                                        rmm::cuda_stream_view stream = cudf::get_default_stream(),
                                                        rmm::device_async_resource_ref = cudf::get_current_device_resource_ref())
{
  b2_column* out = nullptr;
  detail::check(b2_normalize_nans_and_zeros(&input.native(), stream.value(), &out));
  return std::make_unique<column>(out);
}
inline void normalize_nans_and_zeros(mutable_column_view& in_out, rmm::cuda_stream_view stream = cudf::get_default_stream())
{
  detail::check(b2_normalize_nans_and_zeros_inplace(&in_out.native(), stream.value()));
}

}  // namespace cudf
