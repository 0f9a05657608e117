// Test-only: what C++ itself says about the types and values of unary_operation and cast, printed for
// tests/test_unary_oracle.py.
//   "s op id v"           whether the reference's dispatcher for op accepts the numeric type (cpp/src/unary/math_ops.cu:
//                         std::is_arithmetic for SIN .. ABS and NOT, std::is_floating_point for RINT, std::is_integral for
//                         BIT_COUNT / BIT_INVERT, std::is_signed or std::is_floating_point for NEGATE), asked of <type_traits>
//   "c from to v"         whether a cast between the two of the 21 fixed-width ids is allowed: neither side a time_point while
//                         the other is arithmetic (cast_ops.cu:129-137), asked of the std::chrono and arithmetic types
//   "f from to ticks out" std::chrono::floor of `ticks` ticks of one chrono unit in another (cast_ops.cu:45-87)
//   "v name value"        the promotion-sensitive values of the integral overloads
#include <chrono>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <initializer_list>
#include <limits>
#include <tuple>
#include <type_traits>

template <int ID, typename T> struct tag { static constexpr int id = ID; using type = T; };
using days_d  = std::chrono::duration<int32_t, std::ratio<86400>>;
using secs_d  = std::chrono::duration<int64_t>;
using ms_d    = std::chrono::duration<int64_t, std::milli>;
using us_d    = std::chrono::duration<int64_t, std::micro>;
using ns_d    = std::chrono::duration<int64_t, std::nano>;
template <typename D> using tp = std::chrono::time_point<std::chrono::system_clock, D>;
using numeric = std::tuple<tag<1, int8_t>, tag<2, int16_t>, tag<3, int32_t>, tag<4, int64_t>, tag<5, uint8_t>, tag<6, uint16_t>,
                           tag<7, uint32_t>, tag<8, uint64_t>, tag<9, float>, tag<10, double>, tag<11, bool>>;
using chrono  = std::tuple<tag<12, tp<days_d>>, tag<13, tp<secs_d>>, tag<14, tp<ms_d>>, tag<15, tp<us_d>>, tag<16, tp<ns_d>>,
                          tag<17, days_d>, tag<18, secs_d>, tag<19, ms_d>, tag<20, us_d>, tag<21, ns_d>>;
using fixed   = decltype(std::tuple_cat(numeric{}, chrono{}));

template <typename T> struct is_time_point : std::false_type {};
template <typename C, typename D> struct is_time_point<std::chrono::time_point<C, D>> : std::true_type {};
template <typename T> struct duration_of { using type = T; };
template <typename C, typename D> struct duration_of<std::chrono::time_point<C, D>> { using type = D; };

template <typename T>
void support_row(int id)
{
  constexpr bool arith = std::is_arithmetic_v<T>, integral = std::is_integral_v<T>, fp = std::is_floating_point_v<T>;
  for (int op = 0; op < 24; ++op) {
    bool v = false;
    if (op <= 18 || op == 22) v = arith;
    else if (op == 19) v = fp;
    else if (op == 20 || op == 21) v = integral;
    else v = std::is_signed_v<T> || fp;  // NEGATE
    std::printf("s %d %d %d\n", op, id, v ? 1 : 0);
  }
}

template <typename F, typename... Ts>
void cast_row(std::tuple<Ts...>*)
{
  ((std::printf("c %d %d %d\n", F::id, Ts::id,
                (is_time_point<typename F::type>::value && std::is_arithmetic_v<typename Ts::type>) ||
                    (std::is_arithmetic_v<typename F::type> && is_time_point<typename Ts::type>::value)
                  ? 0
                  : 1)),
   ...);
}
template <typename... Fs> void cast_rows(std::tuple<Fs...>*) { (cast_row<Fs>((fixed*)nullptr), ...); }

template <typename F, typename T>
void floor_one(long long ticks)
{
  using DF = typename duration_of<typename F::type>::type;
  using DT = typename duration_of<typename T::type>::type;
  // in int64, before the narrowing to the target's rep
  using DT64 = std::chrono::duration<int64_t, typename DT::period>;
  const auto out = std::chrono::floor<DT64>(std::chrono::duration<int64_t, typename DF::period>(ticks));
  std::printf("f %d %d %lld %lld\n", F::id, T::id, ticks, (long long)out.count());
}
template <typename F, typename... Ts>
void floor_row(std::tuple<Ts...>*)
{
  for (long long t : {0LL, 1LL, -1LL, 999LL, -999LL, 1000LL, -1000LL, -1001LL, 86399LL, -86399LL, -86400LL, -86401LL,
                      1234567890123LL, -1234567890123LL, 86400000000001LL, -86400000000001LL})
    (floor_one<F, Ts>(t), ...);
}
template <typename... Fs> void floor_rows(std::tuple<Fs...>*) { (floor_row<Fs>((chrono*)nullptr), ...); }

int main()
{
  std::apply([](auto... t) { (support_row<typename decltype(t)::type>(decltype(t)::id), ...); }, numeric{});
  cast_rows((fixed*)nullptr);
  floor_rows((chrono*)nullptr);
  const double nan = std::numeric_limits<double>::quiet_NaN();
  bool t = true, f = false;
  std::printf("v bit_invert_true %d\n", (int)static_cast<bool>(~t));
  std::printf("v bit_invert_false %d\n", (int)static_cast<bool>(~f));
  std::printf("v not_true %d\n", (int)(!t));
  std::printf("v not_false %d\n", (int)(!f));
  std::printf("v bit_count_true %d\n", (int)__builtin_popcount(static_cast<unsigned char>(t)));
  std::printf("v abs_int8_min %d\n", (int)static_cast<int8_t>(std::abs(std::numeric_limits<int8_t>::min())));
  std::printf("v abs_int16_min %d\n", (int)static_cast<int16_t>(std::abs(std::numeric_limits<int16_t>::min())));
  std::printf("v negate_int8_min %d\n", (int)static_cast<int8_t>(-std::numeric_limits<int8_t>::min()));
  std::printf("v negate_int16_min %d\n", (int)static_cast<int16_t>(-std::numeric_limits<int16_t>::min()));
  std::printf("v not_nan %d\n", (int)(!nan));
  std::printf("v not_neg_zero %d\n", (int)(!(-0.0)));
  std::printf("v bit_count_int8_m1 %d\n", __builtin_popcount(static_cast<uint8_t>(int8_t(-1))));
  std::printf("v bit_count_int8_min %d\n", __builtin_popcount(static_cast<uint8_t>(std::numeric_limits<int8_t>::min())));
  std::printf("v bit_count_int16_m2 %d\n", __builtin_popcount(static_cast<uint16_t>(int16_t(-2))));
  std::printf("v bool_of_nan %d\n", (int)static_cast<bool>(nan));
  std::printf("v bit_invert_uint8_5 %d\n", (int)static_cast<uint8_t>(~uint8_t(5)));
  return 0;
}
