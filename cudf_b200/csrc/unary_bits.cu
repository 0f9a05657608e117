// unary_bits.cu — unary_kernel (unary.cuh) for BIT_COUNT, BIT_INVERT, NOT and NEGATE (generic path), is_nan / is_not_nan
// (vector path), and validity_kernel for is_null / is_valid.
#include "unary.cuh"

namespace b2 {
namespace unary {
namespace {

__global__ void __launch_bounds__(256) validity_kernel(args a, bool want_valid)
{
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  uint8_t* out         = static_cast<uint8_t*>(a.out);
  for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g * 32 < a.n; g += stride) {
    const int64_t r0 = g * 32;
    uint32_t w       = load_mask_word_unaligned(a.mask, a.bit + r0, a.last_word);
    if (!want_valid) w = ~w;
    // 4 bits -> 4 bytes of 0 / 1: bit k moves to bit 8 k (the shifted copies do not overlap)
    uint32_t b[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) b[k] = (((w >> (4 * k)) & 0xfu) * 0x00204081u) & 0x01010101u;
    if (r0 + 32 <= a.n) {
      st_na_v4(out + r0, make_int4((int)b[0], (int)b[1], (int)b[2], (int)b[3]));
      st_na_v4(out + r0 + 16, make_int4((int)b[4], (int)b[5], (int)b[6], (int)b[7]));
    } else {
      for (int64_t k = 0; r0 + k < a.n; ++k) out[r0 + k] = (uint8_t)((w >> k) & 1u);
    }
  }
}

}  // namespace

void launch_bits(int op, const args& a, cudaStream_t stream)
{
  switch (op) {
    case B2_UNARY_BIT_COUNT:
      switch (type_width(a.in_type)) {
        case 1: return launch<bits_fn<B2_UNARY_BIT_COUNT>, uint8_t, rt, rt>(a, stream);
        case 2: return launch<bits_fn<B2_UNARY_BIT_COUNT>, uint16_t, rt, rt>(a, stream);
        case 4: return launch<bits_fn<B2_UNARY_BIT_COUNT>, uint32_t, rt, rt>(a, stream);
        default: return launch<bits_fn<B2_UNARY_BIT_COUNT>, uint64_t, rt, rt>(a, stream);
      }
    case B2_UNARY_BIT_INVERT: return launch<bits_fn<B2_UNARY_BIT_INVERT>, uint64_t, rt, rt>(a, stream);
    case B2_UNARY_NOT: return launch<bits_fn<B2_UNARY_NOT>, double, rt, rt>(a, stream);
    case B2_UNARY_NEGATE:
      if (a.in_type == B2_FLOAT32) return launch<bits_fn<B2_UNARY_NEGATE>, float, rt, rt>(a, stream);
      if (a.in_type == B2_FLOAT64) return launch<bits_fn<B2_UNARY_NEGATE>, double, rt, rt>(a, stream);
      return launch<bits_fn<B2_UNARY_NEGATE>, uint64_t, rt, rt>(a, stream);
    default: B2_FAIL(B2_ERR_LOGIC, "unary_operation: operator outside the bits family");
  }
}

void launch_nan(bool want_nan, const args& a, cudaStream_t stream)
{
  if (a.in_type == B2_FLOAT32) {
    if (want_nan) return launch<nan_fn<true>, float, float, uint8_t>(a, stream);
    return launch<nan_fn<false>, float, float, uint8_t>(a, stream);
  }
  if (want_nan) return launch<nan_fn<true>, double, double, uint8_t>(a, stream);
  return launch<nan_fn<false>, double, double, uint8_t>(a, stream);
}

void launch_validity(bool want_valid, const args& a, cudaStream_t stream)
{
  B2_LAUNCH(validity_kernel, binop::grid_for((a.n + 1023) / 1024), 256, 0, stream, a, want_valid);
}

}  // namespace unary
}  // namespace b2
