// Test-only: what C++ itself says about the types of binary_operation, printed for tests/test_binaryop_oracle.py.
//   "c a b t"      std::common_type_t<A, B> of every pair of the 11 numeric types (cudf type ids)
//   "t o a b t"    std::common_type_t<O, A, B> of every triple
//   "s op o a b v" whether op is defined on std::common_type_t<A, B> (the expression below is well-formed) and its result is
//                  constructible as O (BOOL8 output for the comparison and logical operators): the rule of
//                  cpp/src/binaryop/compiled/util.cpp, asked of the compiler instead of restated.
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <type_traits>
#include <utility>

template <int ID, typename T> struct tag { static constexpr int id = ID; using type = T; };
using ids = std::tuple<tag<1, int8_t>, tag<2, int16_t>, tag<3, int32_t>, tag<4, int64_t>, tag<5, uint8_t>, tag<6, uint16_t>,
                       tag<7, uint32_t>, tag<8, uint64_t>, tag<9, float>, tag<10, double>, tag<11, bool>>;

template <typename T> constexpr int id_of() { return std::is_same_v<T, int8_t> ? 1 : std::is_same_v<T, int16_t> ? 2 : std::is_same_v<T, int32_t> ? 3
  : std::is_same_v<T, int64_t> ? 4 : std::is_same_v<T, uint8_t> ? 5 : std::is_same_v<T, uint16_t> ? 6 : std::is_same_v<T, uint32_t> ? 7
  : std::is_same_v<T, uint64_t> ? 8 : std::is_same_v<T, float> ? 9 : std::is_same_v<T, double> ? 10 : std::is_same_v<T, bool> ? 11 : -1; }

// the expression of each operator, SFINAE-friendly; -1 marks the operators without one here
#define EXPR_OP(NAME, EXPR) struct NAME { template <typename X, typename Y> auto operator()(X x, Y y) -> decltype(EXPR) { return EXPR; } };
EXPR_OP(Add, x + y) EXPR_OP(Sub, x - y) EXPR_OP(Mul, x * y) EXPR_OP(Div, x / y)
EXPR_OP(TrueDiv, double(x) / double(y)) EXPR_OP(Pow, std::pow(double(x), double(y)))
EXPR_OP(Shl, x << y) EXPR_OP(Shr, x >> y) EXPR_OP(And, x & y) EXPR_OP(Or, x | y) EXPR_OP(Xor, x ^ y)
EXPR_OP(LAnd, x && y) EXPR_OP(LOr, x || y) EXPR_OP(Eq, x == y) EXPR_OP(Lt, x < y)
EXPR_OP(Max, x > y ? x : y)
struct IntOnly { template <typename X, typename Y, typename = std::enable_if_t<std::is_integral_v<X> && std::is_integral_v<Y>>> X operator()(X x, Y) { return x; } };
struct Sru { template <typename X, typename Y, typename = std::enable_if_t<std::is_integral_v<X> && !std::is_same_v<X, bool>>> auto operator()(X x, Y y) -> decltype(std::make_unsigned_t<X>(x) >> y) { return std::make_unsigned_t<X>(x) >> y; } };
// FLOOR_DIV, MOD, PMOD, PYMOD: integer expressions for integers, fmod / floor for floats: defined for every numeric type
struct AnyNum { template <typename X, typename Y> X operator()(X x, Y) { return x; } };

template <typename Op, typename O, typename A, typename B>
constexpr int supported(bool bool_out)
{
  using C = std::common_type_t<A, B>;
  if constexpr (!std::is_invocable_v<Op, C, C>) return 0;
  else if (bool_out) return std::is_same_v<O, bool> ? 1 : 0;
  else return std::is_constructible_v<O, std::invoke_result_t<Op, C, C>> ? 1 : 0;
}

template <typename O, typename A, typename B>
void row()
{
  const int o = id_of<O>(), a = id_of<A>(), b = id_of<B>();
  std::printf("t %d %d %d %d\n", o, a, b, id_of<std::common_type_t<O, A, B>>());
  // cudf::binary_operator values
  const int v[34] = {
    supported<Add, O, A, B>(false), supported<Sub, O, A, B>(false), supported<Mul, O, A, B>(false), supported<Div, O, A, B>(false),
    supported<TrueDiv, O, A, B>(false), supported<AnyNum, O, A, B>(false), supported<AnyNum, O, A, B>(false),
    supported<AnyNum, O, A, B>(false), supported<AnyNum, O, A, B>(false), supported<Pow, O, A, B>(false),
    supported<IntOnly, O, A, B>(false), supported<Pow, O, A, B>(false), supported<Pow, O, A, B>(false),
    supported<Shl, O, A, B>(false), supported<Shr, O, A, B>(false), supported<Sru, O, A, B>(false), supported<And, O, A, B>(false),
    supported<Or, O, A, B>(false), supported<Xor, O, A, B>(false), supported<LAnd, O, A, B>(true), supported<LOr, O, A, B>(true),
    supported<Eq, O, A, B>(true), supported<Eq, O, A, B>(true), supported<Lt, O, A, B>(true), supported<Lt, O, A, B>(true),
    supported<Lt, O, A, B>(true), supported<Lt, O, A, B>(true), supported<Eq, O, A, B>(true), supported<Eq, O, A, B>(true),
    supported<Max, O, A, B>(false), supported<Max, O, A, B>(false), 0 /* GENERIC_BINARY */, supported<LAnd, O, A, B>(true),
    supported<LOr, O, A, B>(true)};
  for (int op = 0; op < 34; ++op) std::printf("s %d %d %d %d %d\n", op, o, a, b, v[op]);
}

template <typename O, typename A, typename... Bs> void rows_b(std::tuple<Bs...>*) { (row<O, A, typename Bs::type>(), ...); }
template <typename O, typename... As> void rows_a(std::tuple<As...>*) { (rows_b<O, typename As::type>((ids*)nullptr), ...); }
template <typename... Os> void rows_o(std::tuple<Os...>*) { (rows_a<typename Os::type>((ids*)nullptr), ...); }
template <typename A, typename... Bs> void pairs_b(std::tuple<Bs...>*)
{
  (std::printf("c %d %d %d\n", id_of<A>(), id_of<typename Bs::type>(), id_of<std::common_type_t<A, typename Bs::type>>()), ...);
}
template <typename... As> void pairs(std::tuple<As...>*) { (pairs_b<typename As::type>((ids*)nullptr), ...); }

int main()
{
  pairs((ids*)nullptr);
  rows_o((ids*)nullptr);
  return 0;
}
