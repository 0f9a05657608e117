// unary_cast.cu — unary_kernel (unary.cuh) for cudf::cast: integer <-> float and FLOAT32 <-> FLOAT64 (vector path), chrono unit
// conversions on the storage integers (vector path), and every other numeric pair on the generic path.
#include "unary.cuh"

namespace b2 {
namespace unary {
namespace {

template <typename In, typename Out>
bool try_typed(const args& a, cudaStream_t stream)
{
  if (a.in_type != type_of<In>() || a.out_type != type_of<Out>()) return false;
  launch<cast_fn, In, In, Out>(a, stream);
  return true;
}

template <typename... Ints>
bool try_int_float(const args& a, cudaStream_t stream)
{
  return (... || (try_typed<Ints, float>(a, stream) || try_typed<Ints, double>(a, stream) || try_typed<float, Ints>(a, stream) ||
                  try_typed<double, Ints>(a, stream)));
}

}  // namespace

void launch_cast(const args& a, cudaStream_t stream)
{
  if (a.mul != 0) {  // chrono -> chrono: the storage types are int32 (DAYS) or int64
    const bool in32 = a.in_type == B2_INT32, out32 = a.out_type == B2_INT32;
    if (in32 && out32) return launch<chrono_fn, int64_t, int32_t, int32_t>(a, stream);
    if (in32) return launch<chrono_fn, int64_t, int32_t, int64_t>(a, stream);
    if (out32) return launch<chrono_fn, int64_t, int64_t, int32_t>(a, stream);
    return launch<chrono_fn, int64_t, int64_t, int64_t>(a, stream);
  }
  if (try_int_float<int8_t, int16_t, int32_t, int64_t, uint8_t, uint16_t, uint32_t, uint64_t>(a, stream) ||
      try_typed<float, double>(a, stream) || try_typed<double, float>(a, stream))
    return;
  // every value of the source is exact in C, and a conversion depends on the value only
  if (is_float_id(a.in_type)) return launch<cast_fn, double, rt, rt>(a, stream);
  if (a.in_type == B2_UINT8 || a.in_type == B2_UINT16 || a.in_type == B2_UINT32 || a.in_type == B2_UINT64)
    return launch<cast_fn, uint64_t, rt, rt>(a, stream);
  return launch<cast_fn, int64_t, rt, rt>(a, stream);
}

}  // namespace unary
}  // namespace b2
