// capi.cu — the extern "C" boundary declared in include/cudf_b200.h plus the small runtime behind it
// (thread-local error slot, stream-ordered pool, owning handles, argument validation).
// Host-side dispatch mirrors the reference entry points: cpp/src/sort/sort.cu:22-100,
// cpp/src/sort/stable_sort.cu, cpp/src/copying/gather.cu, cpp/src/bitmask/null_mask.cu.
#include "common.cuh"
#include "device_utils.cuh"

#include <cstdlib>
#include <mutex>

namespace b2 {

std::atomic<uint64_t> g_launch_count{0};

static thread_local std::string tl_error;
void set_last_error(const char* msg) { tl_error = msg ? msg : ""; }

// ---- profiler ------------------------------------------------------------------------------------
std::atomic<int> g_profile_on{0};
namespace {
struct prof_rec { std::string name; cudaEvent_t e0, e1; };
std::mutex g_prof_mu;
std::vector<prof_rec> g_prof;
}  // namespace
prof_scope::prof_scope(const char* n, cudaStream_t stream) : name(n), s(stream)
{
  if (!g_profile_on.load(std::memory_order_relaxed)) return;
  cudaEventCreate(&e0);
  cudaEventCreate(&e1);
  cudaEventRecord(e0, s);
}
prof_scope::~prof_scope()
{
  if (!e0) return;
  cudaEventRecord(e1, s);
  std::lock_guard<std::mutex> lk(g_prof_mu);
  g_prof.push_back({name, e0, e1});
}

// ---- allocator ----------------------------------------------------------------------------------
// Per device, on first allocation: keep freed blocks cached in the stream-ordered pool (like an rmm pool resource).
static void init_pool_once()
{
  static std::atomic<uint64_t> done{0};
  once_per_device(done, [] {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return;
    cudaMemPool_t pool;
    if (cudaDeviceGetDefaultMemPool(&pool, dev) == cudaSuccess) {
      uint64_t thr = UINT64_MAX;
      cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thr);
    }
  });
}

void* dev_alloc(size_t bytes, cudaStream_t stream)
{
  init_pool_once();
  void* p = nullptr;
  cudaError_t e = cudaMallocAsync(&p, bytes, stream);
  if (e != cudaSuccess) {
    cudaGetLastError();
    throw error(B2_ERR_BAD_ALLOC, std::string("device allocation of ") + std::to_string(bytes) +
                                    " bytes failed: " + cudaGetErrorString(e));
  }
  return p;
}
void dev_free(void* p, cudaStream_t stream) noexcept
{
  if (p) cudaFreeAsync(p, stream);
}

column_ptr make_column(int32_t type_id, int32_t size, bool with_mask, cudaStream_t stream)
{
  auto c = std::make_unique<b2_column>();
  c->type_id = type_id;
  c->size    = size;
  const size_t w = type_width(type_id);
  if (size > 0) {
    c->data = dbuf(w * (size_t)size, stream);
    if (with_mask) {
      c->mask = dbuf(bitmask_bytes(size), stream);
      B2_CUDA_TRY(cudaMemsetAsync(c->mask.ptr, 0, c->mask.bytes, stream));
    }
  }
  return c;
}

void validate_column(const b2_column_view& c)
{
  B2_EXPECTS(is_fixed_width(c.type_id), B2_ERR_DATA_TYPE, "only fixed-width column types are supported on this path");
  B2_EXPECTS(c.size >= 0, B2_ERR_LOGIC, "Column size cannot be negative.");
  B2_EXPECTS(c.offset >= 0, B2_ERR_LOGIC, "Invalid offset.");
  B2_EXPECTS(c.size == 0 || c.data != nullptr, B2_ERR_LOGIC, "Null data pointer.");
  B2_EXPECTS(c.null_count <= 0 || c.null_mask != nullptr, B2_ERR_LOGIC, "Invalid null mask.");
  B2_EXPECTS(c.null_count >= 0 && c.null_count <= c.size, B2_ERR_LOGIC, "Invalid null count.");
}

void validate_table(const b2_table_view* t, std::vector<b2_column_view>& cols)
{
  B2_EXPECTS(t != nullptr, B2_ERR_INVALID_ARGUMENT, "null table_view");
  B2_EXPECTS(t->num_columns >= 0 && (t->num_columns == 0 || t->columns != nullptr), B2_ERR_INVALID_ARGUMENT,
             "invalid table_view");
  cols.assign(t->columns, t->columns + t->num_columns);
  for (auto& c : cols) {
    validate_column(c);
    B2_EXPECTS(c.size == cols[0].size, B2_ERR_LOGIC, "Column size mismatch.");
  }
}

}  // namespace b2

int32_t b2_column::resolve_null_count() const
{
  if (null_count >= 0) return null_count;
  unsigned long long h = 0;
  cudaMemcpyAsync(&h, pending.ptr, sizeof(h), cudaMemcpyDeviceToHost, pending_stream);
  cudaStreamSynchronize(pending_stream);
  null_count = pending_is_valid_count ? size - (int32_t)h : (int32_t)h;
  pending.reset();
  return null_count;
}

using namespace b2;

static cudaStream_t S(b2_stream s) { return static_cast<cudaStream_t>(s); }

extern "C" {

const char* b2_last_error(void) { return tl_error.c_str(); }
const char* b2_version(void) { return "cudf_b200 0.1 (sm_90a)"; }
uint64_t b2_kernel_launch_count(void) { return g_launch_count.load(); }
void b2_profile_enable(int32_t on) { g_profile_on.store(on ? 1 : 0); }
void b2_profile_reset(void)
{
  std::lock_guard<std::mutex> lk(g_prof_mu);
  for (auto& r : g_prof) { cudaEventDestroy(r.e0); cudaEventDestroy(r.e1); }
  g_prof.clear();
}
b2_status b2_profile_get(const char* name, double* total_ms, int64_t* launches)
{
  B2_TRY_BEGIN
  B2_EXPECTS(name && total_ms && launches, B2_ERR_INVALID_ARGUMENT, "null argument");
  B2_CUDA_TRY(cudaDeviceSynchronize());
  std::lock_guard<std::mutex> lk(g_prof_mu);
  double t = 0; int64_t c = 0;
  for (auto& r : g_prof) {
    if (r.name != name) continue;
    float ms = 0;
    B2_CUDA_TRY(cudaEventElapsedTime(&ms, r.e0, r.e1));
    t += ms; ++c;
  }
  *total_ms = t; *launches = c;
  B2_TRY_END
}
b2_status b2_profile_get_over(const char* name, double min_ms, double* total_ms, int64_t* launches)
{
  B2_TRY_BEGIN
  B2_EXPECTS(name && total_ms && launches, B2_ERR_INVALID_ARGUMENT, "null argument");
  B2_CUDA_TRY(cudaDeviceSynchronize());
  std::lock_guard<std::mutex> lk(g_prof_mu);
  double t = 0; int64_t c = 0;
  for (auto& r : g_prof) {
    if (r.name != name) continue;
    float ms = 0;
    B2_CUDA_TRY(cudaEventElapsedTime(&ms, r.e0, r.e1));
    if (ms < min_ms) continue;
    t += ms; ++c;
  }
  *total_ms = t; *launches = c;
  B2_TRY_END
}
b2_status b2_trim_pool(void)
{
  B2_TRY_BEGIN
  int dev = 0;
  B2_CUDA_TRY(cudaGetDevice(&dev));
  cudaMemPool_t pool;
  B2_CUDA_TRY(cudaDeviceGetDefaultMemPool(&pool, dev));
  B2_CUDA_TRY(cudaDeviceSynchronize());
  B2_CUDA_TRY(cudaMemPoolTrimTo(pool, 0));
  B2_TRY_END
}

// ---- handles ------------------------------------------------------------------------------------
b2_status b2_column_view_of(const b2_column* col, b2_column_view* out)
{
  B2_TRY_BEGIN
  B2_EXPECTS(col && out, B2_ERR_INVALID_ARGUMENT, "null argument");
  *out = col->view();
  B2_TRY_END
}
void b2_column_free(b2_column* col) { delete col; }
int32_t b2_table_num_columns(const b2_table* t) { return t ? (int32_t)t->cols.size() : 0; }
int32_t b2_table_num_rows(const b2_table* t) { return (t && !t->cols.empty()) ? t->cols[0]->size : 0; }
const b2_column* b2_table_column(const b2_table* t, int32_t i)
{
  return (t && i >= 0 && i < (int32_t)t->cols.size()) ? t->cols[i].get() : nullptr;
}
b2_status b2_table_release(b2_table* t, b2_column** out_cols, int32_t capacity)
{
  B2_TRY_BEGIN
  B2_EXPECTS(t && out_cols, B2_ERR_INVALID_ARGUMENT, "null argument");
  B2_EXPECTS(capacity >= (int32_t)t->cols.size(), B2_ERR_INVALID_ARGUMENT, "capacity too small");
  for (size_t i = 0; i < t->cols.size(); ++i) out_cols[i] = t->cols[i].release();
  t->cols.clear();
  B2_TRY_END
}
void b2_table_free(b2_table* t) { delete t; }
void* b2_buffer_data(const b2_buffer* b) { return b ? b->buf.ptr : nullptr; }
size_t b2_buffer_size(const b2_buffer* b) { return b ? b->buf.bytes : 0; }
void b2_buffer_free(b2_buffer* b) { delete b; }

b2_status b2_scalar_create(int32_t type_id, const void* host_value, int32_t is_valid, b2_stream stream, b2_scalar** out)
{
  B2_TRY_BEGIN
  B2_EXPECTS(out, B2_ERR_INVALID_ARGUMENT, "null argument");
  *out = make_scalar(type_id, host_value, is_valid != 0, S(stream)).release();
  B2_TRY_END
}
int32_t b2_scalar_type(const b2_scalar* s) { return s ? s->type_id : B2_EMPTY; }
const void* b2_scalar_device_data(const b2_scalar* s) { return s ? s->data.ptr : nullptr; }
b2_status b2_scalar_get(const b2_scalar* s, b2_stream stream, void* host_value, int32_t* is_valid)
{
  B2_TRY_BEGIN
  B2_EXPECTS(s, B2_ERR_INVALID_ARGUMENT, "null scalar");
  unsigned char h[16] = {0};
  B2_CUDA_TRY(cudaMemcpyAsync(h, s->data.ptr, 12, cudaMemcpyDeviceToHost, S(stream)));
  B2_CUDA_TRY(cudaStreamSynchronize(S(stream)));
  if (host_value) memcpy(host_value, h, 8);
  if (is_valid) {
    int32_t v;
    memcpy(&v, h + 8, 4);
    *is_valid = v != 0;
  }
  B2_TRY_END
}
void b2_scalar_free(b2_scalar* s) { delete s; }

// ---- null masks ---------------------------------------------------------------------------------
size_t b2_bitmask_allocation_size_bytes(int32_t bits) { return bitmask_bytes(bits); }

b2_status b2_create_null_mask(int32_t size, int32_t state, b2_stream stream, b2_buffer** out)
{
  B2_TRY_BEGIN
  B2_EXPECTS(out, B2_ERR_INVALID_ARGUMENT, "null argument");
  B2_EXPECTS(size >= 0, B2_ERR_LOGIC, "Invalid size.");
  auto b = std::make_unique<b2_buffer>();
  if (state != B2_MASK_UNALLOCATED && size > 0) {
    b->buf = dbuf(bitmask_bytes(size), S(stream));
    if (state != B2_MASK_UNINITIALIZED)
      B2_CUDA_TRY(cudaMemsetAsync(b->buf.ptr, state == B2_MASK_ALL_VALID ? 0xff : 0x00, b->buf.bytes, S(stream)));
  }
  *out = b.release();
  B2_TRY_END
}
b2_status b2_set_null_mask(uint32_t* bitmask, int32_t begin, int32_t end, int32_t valid, b2_stream stream)
{
  B2_TRY_BEGIN
  set_null_mask(bitmask, begin, end, valid != 0, S(stream));
  B2_TRY_END
}
b2_status b2_copy_bitmask(const uint32_t* mask, int32_t begin, int32_t end, b2_stream stream, b2_buffer** out)
{
  B2_TRY_BEGIN
  B2_EXPECTS(out, B2_ERR_INVALID_ARGUMENT, "null argument");
  auto b = std::make_unique<b2_buffer>();
  b->buf = copy_bitmask(mask, begin, end, S(stream));
  *out = b.release();
  B2_TRY_END
}
b2_status b2_count_set_bits(const uint32_t* bitmask, int32_t start, int32_t stop, b2_stream stream, int32_t* out)
{
  B2_TRY_BEGIN
  B2_EXPECTS(out, B2_ERR_INVALID_ARGUMENT, "null argument");
  *out = count_set_bits(bitmask, start, stop, S(stream));
  B2_TRY_END
}
b2_status b2_null_count(const uint32_t* bitmask, int32_t start, int32_t stop, b2_stream stream, int32_t* out)
{
  B2_TRY_BEGIN
  B2_EXPECTS(out, B2_ERR_INVALID_ARGUMENT, "null argument");
  B2_EXPECTS(start >= 0 && start <= stop, B2_ERR_LOGIC, "Invalid bit range.");
  *out = bitmask == nullptr ? 0 : (stop - start) - count_set_bits(bitmask, start, stop, S(stream));
  B2_TRY_END
}
b2_status b2_bitmask_and(const b2_table_view* view, b2_stream stream, b2_buffer** out_mask, int32_t* out_null_count)
{
  B2_TRY_BEGIN
  B2_EXPECTS(out_mask && out_null_count, B2_ERR_INVALID_ARGUMENT, "null argument");
  std::vector<b2_column_view> cols;
  validate_table(view, cols);
  auto b = std::make_unique<b2_buffer>();
  b->buf = bitmask_and(cols, cols.empty() ? 0 : cols[0].size, out_null_count, S(stream));
  *out_mask = b.release();
  B2_TRY_END
}

// ---- gather -------------------------------------------------------------------------------------
b2_status b2_gather(const b2_table_view* source, const b2_column_view* gather_map, int32_t oob_policy, b2_stream stream,
                    b2_table** out)
{
  B2_TRY_BEGIN
  B2_EXPECTS(gather_map && out, B2_ERR_INVALID_ARGUMENT, "null argument");
  std::vector<b2_column_view> cols;
  validate_table(source, cols);
  B2_EXPECTS(!has_nulls(*gather_map), B2_ERR_INVALID_ARGUMENT, "gather_map contains nulls");
  B2_EXPECTS(gather_map->type_id == B2_INT32 || gather_map->type_id == B2_UINT32 || gather_map->size == 0, B2_ERR_DATA_TYPE,
             "gather_map must be INT32 (size_type) on this path");
  const int32_t* map = static_cast<const int32_t*>(gather_map->data) + gather_map->offset;
  *out = gather_table(cols, map, gather_map->size, oob_policy == B2_OOB_NULLIFY, S(stream)).release();
  B2_TRY_END
}

// ---- sort ---------------------------------------------------------------------------------------
b2_status b2_sorted_order(const b2_table_view* keys, const uint8_t* column_order, int32_t n_order,
                          const uint8_t* null_precedence, int32_t n_null_prec, int32_t stable, b2_stream stream,
                          b2_column** out)
{
  B2_TRY_BEGIN
  B2_EXPECTS(out, B2_ERR_INVALID_ARGUMENT, "null argument");
  std::vector<b2_column_view> cols;
  validate_table(keys, cols);
  *out = sorted_order(cols, vec_u8(column_order, n_order), vec_u8(null_precedence, n_null_prec), stable != 0, S(stream))
           .release();
  B2_TRY_END
}

// cudf::detail::sort_by_key — cpp/src/sort/sort.cu:31-50 (stable twin: stable_sort.cu)
static table_ptr sort_by_key_impl(const std::vector<b2_column_view>& values, const std::vector<b2_column_view>& keys,
                                  const std::vector<uint8_t>& order, const std::vector<uint8_t>& nprec, bool stable,
                                  cudaStream_t stream)
{
  const int32_t vrows = values.empty() ? 0 : values[0].size;
  const int32_t krows = keys.empty() ? 0 : keys[0].size;
  B2_EXPECTS(vrows == krows, B2_ERR_LOGIC, "Mismatch in number of rows for values and keys");
  if (keys.size() == 1 && values.size() == 1 && order.size() <= 1 && nprec.size() <= 1) {
    const bool asc = order.empty() ? true : order[0] == B2_ASCENDING;
    if (sort_carry_applicable(keys[0], values[0], asc)) {  // single fixed-width payload: carried through the passes
      auto t = std::make_unique<b2_table>();
      t->cols.push_back(sort_by_key_carry(keys[0], values[0], asc, stream));
      return t;
    }
  }
  auto order_col = sorted_order(keys, order, nprec, stable, stream);
  return gather_table(values, order_col->data.as<int32_t>(), order_col->size, false, stream);
}

b2_status b2_sort(const b2_table_view* input, const uint8_t* column_order, int32_t n_order, const uint8_t* null_precedence,
                  int32_t n_null_prec, int32_t stable, b2_stream stream, b2_table** out)
{
  B2_TRY_BEGIN
  B2_EXPECTS(out, B2_ERR_INVALID_ARGUMENT, "null argument");
  std::vector<b2_column_view> cols;
  validate_table(input, cols);
  auto order = vec_u8(column_order, n_order);
  auto nprec = vec_u8(null_precedence, n_null_prec);
  // fast path: single fixed-width column without nulls -> keys-only radix (sort.cu:58-65)
  if (cols.size() == 1 && is_radix_sortable(cols[0]) && !is_float_id(cols[0].type_id)) {
    B2_EXPECTS(order.size() <= 1 && nprec.size() <= 1, B2_ERR_LOGIC, "Mismatch between number of columns and column order.");
    const bool asc = order.empty() ? true : order[0] == B2_ASCENDING;
    auto t = std::make_unique<b2_table>();
    t->cols.push_back(sort_single_column(cols[0], asc, S(stream)));
    *out = t.release();
  } else {
    *out = sort_by_key_impl(cols, cols, order, nprec, stable != 0, S(stream)).release();
  }
  B2_TRY_END
}

b2_status b2_sort_by_key(const b2_table_view* values, const b2_table_view* keys, const uint8_t* column_order, int32_t n_order,
                         const uint8_t* null_precedence, int32_t n_null_prec, int32_t stable, b2_stream stream,
                         b2_table** out)
{
  B2_TRY_BEGIN
  B2_EXPECTS(out, B2_ERR_INVALID_ARGUMENT, "null argument");
  std::vector<b2_column_view> vcols, kcols;
  validate_table(values, vcols);
  validate_table(keys, kcols);
  *out = sort_by_key_impl(vcols, kcols, vec_u8(column_order, n_order), vec_u8(null_precedence, n_null_prec), stable != 0,
                          S(stream))
           .release();
  B2_TRY_END
}

// ---- reduce / scan / segmented reduce ----------------------------------------------------------
b2_status b2_reduce(const b2_column_view* col, int32_t agg_kind, int32_t output_type_id, const b2_scalar* init, b2_stream stream,
                    b2_scalar** out)
{
  B2_TRY_BEGIN
  B2_EXPECTS(col && out, B2_ERR_INVALID_ARGUMENT, "null argument");
  *out = reduce(*col, agg_kind, output_type_id, init, S(stream)).release();
  B2_TRY_END
}
b2_status b2_segmented_reduce(const b2_column_view* values, const int32_t* offsets, int32_t num_offsets, int32_t agg_kind,
                              int32_t output_type_id, int32_t null_handling, const b2_scalar* init, b2_stream stream,
                              b2_column** out)
{
  B2_TRY_BEGIN
  B2_EXPECTS(values && out, B2_ERR_INVALID_ARGUMENT, "null argument");
  *out = segmented_reduce(*values, offsets, num_offsets, agg_kind, output_type_id, null_handling, init, S(stream)).release();
  B2_TRY_END
}
b2_status b2_scan(const b2_column_view* col, int32_t agg_kind, int32_t scan_type, int32_t null_handling, b2_stream stream,
                  b2_column** out)
{
  B2_TRY_BEGIN
  B2_EXPECTS(col && out, B2_ERR_INVALID_ARGUMENT, "null argument");
  *out = scan(*col, agg_kind, scan_type, null_handling, S(stream)).release();
  B2_TRY_END
}

}  // extern "C"
