// key_pack.cuh — packs the key columns of a row into 64 bits + a per-column null bitmap, normalised so
// that bit equality is the reference's row equality for fixed-width keys (-0 == +0, NaN == NaN:
// cpp/include/cudf/detail/row_operator/primitive_row_operators.cuh:121-143, common_utils.cuh:214-220).
// Shared by the hash join and the hash groupby.
#pragma once
#include "common.cuh"
#include "device_utils.cuh"

namespace b2 {

constexpr int MAX_KEY_COLS = 8;

struct key_cols {
  const void* data[MAX_KEY_COLS];
  const uint32_t* mask[MAX_KEY_COLS];
  int32_t offset[MAX_KEY_COLS];
  int8_t width[MAX_KEY_COLS];
  int8_t is_float[MAX_KEY_COLS];
  int32_t n;
};

struct alignas(16) slot_t {
  uint64_t key;
  int32_t row;
  uint32_t nullbits;
};

__device__ __forceinline__ void pack_row(const key_cols& kc, int64_t r, uint64_t& key, uint32_t& nullbits)
{
  key = 0;
  nullbits = 0;
  int sh = 0;
#pragma unroll 1
  for (int c = 0; c < kc.n; ++c) {
    const int w = kc.width[c];
    const int64_t e = r + kc.offset[c];
    uint64_t bits = 0;
    const bool valid = kc.mask[c] == nullptr || bit_is_set(kc.mask[c], e);
    if (valid) {
      switch (w) {
        case 1: bits = __ldcs(static_cast<const uint8_t*>(kc.data[c]) + e); break;  // streamed once: evict-first
        case 2: bits = __ldcs(static_cast<const uint16_t*>(kc.data[c]) + e); break;
        case 4: {
          uint32_t b = __ldcs(static_cast<const uint32_t*>(kc.data[c]) + e);
          if (kc.is_float[c]) {
            if ((b << 1) == 0) b = 0;                                // -0 -> +0
            else if ((b & 0x7fffffffu) > 0x7f800000u) b = 0x7fc00000u;  // canonical NaN
          }
          bits = b;
          break;
        }
        default: {
          uint64_t b = __ldcs(reinterpret_cast<const unsigned long long*>(kc.data[c]) + e);
          if (kc.is_float[c]) {
            if ((b << 1) == 0) b = 0;
            else if ((b & 0x7fffffffffffffffull) > 0x7ff0000000000000ull) b = 0x7ff8000000000000ull;
          }
          bits = b;
        }
      }
    } else {
      nullbits |= 1u << c;
    }
    key |= bits << sh;
    sh += 8 * w;
  }
}


// ---- wide keys (sum of the key column widths > 8 bytes) -------------------------------------------
// The table stores a 64-bit HASH of the row instead of the packed key; hash equality is then confirmed by
// comparing the key columns of the two rows (the slot's representative / build row against the probing row).
// Same normalisation as pack_row, so the row equality is the reference's (primitive_row_operators.cuh:121-143).
__device__ __forceinline__ uint64_t key_col_bits(const key_cols& kc, int c, int64_t e)
{
  switch (kc.width[c]) {
    case 1: return static_cast<const uint8_t*>(kc.data[c])[e];
    case 2: return static_cast<const uint16_t*>(kc.data[c])[e];
    case 4: {
      uint32_t b = static_cast<const uint32_t*>(kc.data[c])[e];
      if (kc.is_float[c]) {
        if ((b << 1) == 0) b = 0;
        else if ((b & 0x7fffffffu) > 0x7f800000u) b = 0x7fc00000u;
      }
      return b;
    }
    default: {
      uint64_t b = static_cast<const uint64_t*>(kc.data[c])[e];
      if (kc.is_float[c]) {
        if ((b << 1) == 0) b = 0;
        else if ((b & 0x7fffffffffffffffull) > 0x7ff0000000000000ull) b = 0x7ff8000000000000ull;
      }
      return b;
    }
  }
}

__device__ __forceinline__ void hash_row_wide(const key_cols& kc, int64_t r, uint64_t& h, uint32_t& nullbits)
{
  h = 0x9E3779B97F4A7C15ull;
  nullbits = 0;
#pragma unroll 1
  for (int c = 0; c < kc.n; ++c) {
    const int64_t e = r + kc.offset[c];
    uint64_t bits = 0;
    if (kc.mask[c] == nullptr || bit_is_set(kc.mask[c], e)) bits = key_col_bits(kc, c, e);
    else nullbits |= 1u << c;
    h = mix64(h ^ bits) + (uint64_t)c;
  }
}

// row ra of table a == row rb of table b (null == null: callers skip rows with nulls when nulls compare unequal)
__device__ __forceinline__ bool rows_equal_wide(const key_cols& a, int64_t ra, const key_cols& b, int64_t rb)
{
#pragma unroll 1
  for (int c = 0; c < a.n; ++c) {
    const int64_t ea = ra + a.offset[c], eb = rb + b.offset[c];
    const bool va = a.mask[c] == nullptr || bit_is_set(a.mask[c], ea);
    const bool vb = b.mask[c] == nullptr || bit_is_set(b.mask[c], eb);
    if (va != vb) return false;
    if (va && key_col_bits(a, c, ea) != key_col_bits(b, c, eb)) return false;
  }
  return true;
}

__device__ __forceinline__ uint32_t slot_hash(uint64_t key, uint32_t nullbits, uint32_t mask)
{
  return (uint32_t)mix64(key + 0x9E3779B97F4A7C15ull * (nullbits + 1)) & mask;
}

__device__ __forceinline__ slot_t load_slot(const slot_t* p)
{
  int4 v = *reinterpret_cast<const int4*>(p);
  slot_t s;
  memcpy(&s, &v, 16);
  return s;
}

__device__ __forceinline__ slot_t cas128(slot_t* addr, const slot_t& expected, const slot_t& desired)
{
  uint64_t e0, e1, d0, d1, r0, r1;
  memcpy(&e0, &expected, 8);
  memcpy(&e1, reinterpret_cast<const char*>(&expected) + 8, 8);
  memcpy(&d0, &desired, 8);
  memcpy(&d1, reinterpret_cast<const char*>(&desired) + 8, 8);
#ifdef B2_EMU
  memcpy(&r0, addr, 8);
  memcpy(&r1, reinterpret_cast<const char*>(addr) + 8, 8);
  if (r0 == e0 && r1 == e1) {
    memcpy(addr, &d0, 8);
    memcpy(reinterpret_cast<char*>(addr) + 8, &d1, 8);
  }
#else
  asm volatile(
    "{\n .reg .b128 e, d, r;\n mov.b128 e, {%2, %3};\n mov.b128 d, {%4, %5};\n"
    " atom.global.cas.b128 r, [%6], e, d;\n mov.b128 {%0, %1}, r;\n}"
    : "=l"(r0), "=l"(r1)
    : "l"(e0), "l"(e1), "l"(d0), "l"(d1), "l"(addr)
    : "memory");
#endif
  slot_t out;
  memcpy(&out, &r0, 8);
  memcpy(reinterpret_cast<char*>(&out) + 8, &r1, 8);
  return out;
}

__device__ __forceinline__ slot_t load_slot_volatile(const slot_t* p)
{
#ifdef B2_EMU
  const uint4 v = *reinterpret_cast<const uint4*>(p);
#else
  uint4 v;
  asm volatile("ld.volatile.global.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p) : "memory");
#endif
  slot_t s;
  memcpy(&s, &v, 16);
  return s;
}

inline int key_bytes(const std::vector<b2_column_view>& cols)
{
  int total = 0;
  for (const auto& v : cols) total += type_width(v.type_id);
  return total;
}
inline bool keys_are_wide(const std::vector<b2_column_view>& cols) { return key_bytes(cols) > 8; }

inline key_cols make_key_cols(const std::vector<b2_column_view>& cols, bool allow_wide = false)
{
  B2_EXPECTS(cols.size() <= (size_t)MAX_KEY_COLS, B2_ERR_INVALID_ARGUMENT, "at most 8 key columns are supported on this path");
  key_cols kc{};
  int total = 0;
  for (size_t c = 0; c < cols.size(); ++c) {
    const auto& v = cols[c];
    kc.data[c]     = v.data;
    kc.mask[c]     = has_nulls(v) ? v.null_mask : nullptr;
    kc.offset[c]   = v.offset;
    kc.width[c]    = (int8_t)type_width(v.type_id);
    kc.is_float[c] = is_float_id(v.type_id) ? 1 : 0;
    total += kc.width[c];
  }
  kc.n = (int32_t)cols.size();
  for (const auto& v : cols) B2_EXPECTS(is_fixed_width(v.type_id), B2_ERR_DATA_TYPE, "key columns must be fixed-width");
  B2_EXPECTS(allow_wide || total <= 8, B2_ERR_INVALID_ARGUMENT,
             "the packed key (sum of key column widths) must fit in 8 bytes on this path");
  return kc;
}


}  // namespace b2
