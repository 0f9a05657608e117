"""Known answers of the reference's unary tests, transcribed as data: cpp/tests/unary/math_ops_test.cpp, unary_ops_test.cpp and
the non-decimal cases of cast_tests.cpp.

A case: {"src", "fn": unary | cast | is_null | is_valid | is_nan | is_not_nan, "type": input type id, "values", "valid" (None:
no mask), "op" (unary), "to" (cast; a list: casts in order), and "expect" (output values, None at null rows) with "expect_type", or "raises": the
exception class name}. "approx": a libm result, compared within 4 ulp. Typed tests (TYPED_TEST) appear once per type of their type list."""
NAN = float("nan")
INF = float("inf")
INT8, INT16, INT32, INT64, UINT8, UINT16, UINT32, UINT64, FLOAT32, FLOAT64, BOOL8 = range(1, 12)
NUMERIC = list(range(1, 12))            # cudf::test::NumericTypes
INTEGRAL_NOT_BOOL = list(range(1, 9))   # cudf::test::IntegralTypesNotBool
FLOATS = [FLOAT32, FLOAT64]
TS_D, TS_S, TS_MS, TS_US, TS_NS, DUR_D, DUR_S, DUR_MS, DUR_US, DUR_NS = range(12, 22)
(SIN, COS, TAN, ARCSIN, ARCCOS, ARCTAN, SINH, COSH, TANH, ARCSINH, ARCCOSH, ARCTANH, EXP, LOG, SQRT, CBRT, CEIL, FLOOR, ABS, RINT,
 BIT_COUNT, BIT_INVERT, NOT, NEGATE) = range(24)

CASES = []


def _add(**c):
    c.setdefault("valid", None)
    CASES.append(c)


def _popcount_unsigned(v, t):
    bits = {INT8: 8, INT16: 16, INT32: 32, INT64: 64, UINT8: 8, UINT16: 16, UINT32: 32, UINT64: 64}[t]
    return bin(v % (1 << bits)).count("1")


# ---- math_ops_test.cpp -------------------------------------------------------------------------------------------------
# UnaryNegateTests::SimpleNEGATE over the signed integers, floats and durations
for t in [INT8, INT16, INT32, INT64, FLOAT32, FLOAT64, DUR_D, DUR_S, DUR_MS, DUR_US, DUR_NS]:
    _add(src="math_ops_test.cpp:37 SimpleNEGATE", fn="unary", op=NEGATE, type=t, values=[0, 1, 2, 3], expect=[0, -1, -2, -3],
         expect_type=t)
# UnaryNegateErrorTests::UnsupportedTypesFail: unsigned integers, bool, timestamps
for t in [UINT8, UINT16, UINT32, UINT64, BOOL8, TS_D, TS_S, TS_MS, TS_US, TS_NS]:
    _add(src="math_ops_test.cpp:62 NegateUnsupportedTypesFail", fn="unary", op=NEGATE, type=t, values=[1, 2, 3, 4],
         raises="RuntimeError")
# BitCountBool
_b = [True, False, True, True, False, True, False, False]
_add(src="math_ops_test.cpp:89 BitCountBool", fn="unary", op=BIT_COUNT, type=BOOL8, values=_b, expect=[int(x) for x in _b],
     expect_type=INT32)
# BitCount / BitCountWithNulls: 1 .. 15
for t in INTEGRAL_NOT_BOOL:
    _v = list(range(1, 16))
    _add(src="math_ops_test.cpp:105 BitCount", fn="unary", op=BIT_COUNT, type=t, values=_v,
         expect=[_popcount_unsigned(x, t) for x in _v], expect_type=INT32)
    _valid = [i not in (2, 5, 9, 12) for i in range(15)]
    _add(src="math_ops_test.cpp:128 BitCountWithNulls", fn="unary", op=BIT_COUNT, type=t, values=_v, valid=_valid,
         expect=[_popcount_unsigned(x, t) if ok else None for x, ok in zip(_v, _valid)], expect_type=INT32)
for t in NUMERIC:
    # LogicalNot: 1 .. 5 (nonzero) -> false; SimpleLogicalNot; SimpleLogicalNotWithNullMask; EmptyLogicalNot
    _add(src="math_ops_test.cpp:158 LogicalNot", fn="unary", op=NOT, type=t, values=[1, 1, 1, 0, 1] if t == BOOL8 else [1, 2, 3, 0, 5],
         expect=[False, False, False, True, False], expect_type=BOOL8)
    _add(src="math_ops_test.cpp:179 SimpleLogicalNot", fn="unary", op=NOT, type=t, values=[1, 1, 1, 1],
         expect=[False, False, False, False], expect_type=BOOL8)
    _add(src="math_ops_test.cpp:190 SimpleLogicalNotWithNullMask", fn="unary", op=NOT, type=t, values=[1, 1, 1, 1],
         valid=[True, False, True, True], expect=[False, None, False, False], expect_type=BOOL8)
    _add(src="math_ops_test.cpp:202 EmptyLogicalNot", fn="unary", op=NOT, type=t, values=[], expect=[], expect_type=BOOL8)
    # SimpleABS (bool and unsigned: the values as they are), SimpleSQRT, SimpleCBRT and their null-mask and empty forms
    if t == BOOL8:
        _add(src="math_ops_test.cpp:267 SimpleABS", fn="unary", op=ABS, type=t, values=[1, 1, 1, 1], expect=[True] * 4,
             expect_type=t)
    elif t in (INT8, INT16, INT32, INT64, FLOAT32, FLOAT64):
        _add(src="math_ops_test.cpp:267 SimpleABS", fn="unary", op=ABS, type=t, values=[-2, -1, 1, 2], expect=[2, 1, 1, 2],
             expect_type=t)
    else:
        _add(src="math_ops_test.cpp:267 SimpleABS", fn="unary", op=ABS, type=t, values=[2, 1, 1, 2], expect=[2, 1, 1, 2],
             expect_type=t)
    if t != BOOL8:
        _add(src="math_ops_test.cpp:276 SimpleSQRT", fn="unary", op=SQRT, type=t, values=[1, 4, 9, 16], expect=[1, 2, 3, 4],
             expect_type=t)
        _add(src="math_ops_test.cpp:284 SimpleCBRT", fn="unary", op=CBRT, type=t, values=[1, 27, 125], expect=[1, 3, 5],
             expect_type=t, approx=t in FLOATS)
        _add(src="math_ops_test.cpp:292 SimpleSQRTWithNullMask", fn="unary", op=SQRT, type=t, values=[1, 4, 9, 16],
             valid=[True, True, False, True], expect=[1, 2, None, 4], expect_type=t)
        _add(src="math_ops_test.cpp:300 SimpleCBRTWithNullMask", fn="unary", op=CBRT, type=t, values=[1, 27, 125],
             valid=[True, True, False], expect=[1, 3, None], expect_type=t, approx=t in FLOATS)
    _add(src="math_ops_test.cpp:308 EmptyABS", fn="unary", op=ABS, type=t, values=[], expect=[], expect_type=t)
    _add(src="math_ops_test.cpp:316 EmptySQRT", fn="unary", op=SQRT, type=t, values=[], expect=[], expect_type=t)
for t in FLOATS:
    for op, x, e in [(SIN, 0.0, 0.0), (COS, 0.0, 1.0), (TAN, 0.0, 0.0), (ARCSIN, 0.0, 0.0), (ARCCOS, 1.0, 0.0), (ARCTAN, 0.0, 0.0),
                     (SINH, 0.0, 0.0), (COSH, 0.0, 1.0), (TANH, 0.0, 0.0), (ARCSINH, 0.0, 0.0), (ARCCOSH, 1.0, 0.0),
                     (ARCTANH, 0.0, 0.0)]:
        _add(src="math_ops_test.cpp:362-440 Simple" + ["SIN", "COS", "TAN", "ASIN", "ACOS", "ATAN", "SINH", "COSH", "TANH", "ASINH",
                                                       "ACOSH", "ATANH"][op], fn="unary", op=op, type=t, values=[x], expect=[e],
             expect_type=t)
    _add(src="math_ops_test.cpp:442 SimpleFLOOR", fn="unary", op=FLOOR, type=t, values=[1.1, 3.3, 5.5, 7.7], expect=[1.0, 3.0, 5.0, 7.0],
         expect_type=t)
    _add(src="math_ops_test.cpp:450 SimpleCEIL", fn="unary", op=CEIL, type=t, values=[1.1, 3.3, 5.5, 7.7], expect=[2.0, 4.0, 6.0, 8.0],
         expect_type=t)
    _add(src="math_ops_test.cpp:458 SimpleRINT", fn="unary", op=RINT, type=t, values=[1.5, 3.5, -1.5, -3.5, 0.0, NAN],
         expect=[2.0, 4.0, -2.0, -4.0, 0.0, NAN], expect_type=t)
    # SimpleEXP / SimpleLOG: the expected values are std::exp / std::log of the inputs ("approx": within 4 ulp)
    _add(src="math_ops_test.cpp:469 SimpleEXP", fn="unary", op=EXP, type=t, values=[1.5, 3.5, -1.5, -3.5, 0.0, NAN],
         expect=[4.4816890703380645, 33.11545195869231, 0.22313016014842982, 0.0301973834223185, 1.0, NAN], expect_type=t,
         approx=True)
    _add(src="math_ops_test.cpp:482 SimpleLOG", fn="unary", op=LOG, type=t, values=[1.5, 3.5, 1.0, INF, 0.0, NAN, -1.0],
         expect=[0.4054651081081644, 1.252762968495368, 0.0, INF, -INF, NAN, NAN], expect_type=t, approx=True)
# RINTNonFloatingFail, IntegralTypeFail (BIT_INVERT on floats), ArithmeticTypeFail (math operators on chrono types)
for t in [INT8, INT16, INT32, INT64, UINT8, UINT16, UINT32, UINT64, BOOL8]:
    _add(src="math_ops_test.cpp RINTNonFloatingFail", fn="unary", op=RINT, type=t, values=[1, 2, 3], raises="RuntimeError")
for t in FLOATS:
    _add(src="math_ops_test.cpp IntegralTypeFail", fn="unary", op=BIT_INVERT, type=t, values=[1.0], raises="RuntimeError")
for t in [TS_D, TS_S, TS_MS, TS_US, TS_NS, DUR_D, DUR_NS]:
    _add(src="math_ops_test.cpp ArithmeticTypeFail", fn="unary", op=SQRT, type=t, values=[1], raises="RuntimeError")

# ---- unary_ops_test.cpp ------------------------------------------------------------------------------------------------
for t in NUMERIC:
    _v = [5, 4, 3, 2, 1, 0] if t != BOOL8 else [1, 1, 1, 1, 1, 0]
    _add(src="unary_ops_test.cpp:54 IsNull AllValid", fn="is_null", type=t, values=_v, expect=[False] * 6, expect_type=BOOL8)
    _add(src="unary_ops_test.cpp:69 IsNull WithInvalids", fn="is_null", type=t, values=_v,
         valid=[True, False, True, False, True, False], expect=[False, True, False, True, False, True], expect_type=BOOL8)
    _add(src="unary_ops_test.cpp:84 IsNull EmptyColumns", fn="is_null", type=t, values=[], expect=[], expect_type=BOOL8)
    _add(src="unary_ops_test.cpp:104 IsNotNull AllValid", fn="is_valid", type=t, values=_v, expect=[True] * 6, expect_type=BOOL8)
    _add(src="unary_ops_test.cpp:119 IsNotNull WithInvalids", fn="is_valid", type=t, values=_v,
         valid=[True, False, True, False, True, False], expect=[True, False, True, False, True, False], expect_type=BOOL8)
    _add(src="unary_ops_test.cpp:134 IsNotNull EmptyColumns", fn="is_valid", type=t, values=[], expect=[], expect_type=BOOL8)
for t in FLOATS:
    _v = [1.0, 2.0, NAN, 4.0, NAN, 6.0, 7.0]
    _m = [True, False, True, True, False, True, True]
    _add(src="unary_ops_test.cpp:154 IsNAN AllValid", fn="is_nan", type=t, values=_v,
         expect=[False, False, True, False, True, False, False], expect_type=BOOL8)
    _add(src="unary_ops_test.cpp:167 IsNAN WithNull", fn="is_nan", type=t, values=_v, valid=_m,
         expect=[False, False, True, False, False, False, False], expect_type=BOOL8)
    _add(src="unary_ops_test.cpp:182 IsNAN EmptyColumn", fn="is_nan", type=t, values=[], expect=[], expect_type=BOOL8)
    _add(src="unary_ops_test.cpp:206 IsNotNAN AllValid", fn="is_not_nan", type=t, values=_v,
         expect=[True, True, False, True, False, True, True], expect_type=BOOL8)
    _add(src="unary_ops_test.cpp:219 IsNotNAN WithNull", fn="is_not_nan", type=t, values=_v, valid=_m,
         expect=[True, True, False, True, True, True, True], expect_type=BOOL8)
    _add(src="unary_ops_test.cpp:234 IsNotNAN EmptyColumn", fn="is_not_nan", type=t, values=[], expect=[], expect_type=BOOL8)
for fn in ("is_nan", "is_not_nan"):
    _add(src="unary_ops_test.cpp:194 NonFloatingColumn", fn=fn, type=INT32, values=[1, 2, 5, 3, 5, 6, 7],
         valid=[True, False, True, True, False, True, True], raises="RuntimeError")

# ---- cast_tests.cpp (non-decimal) --------------------------------------------------------------------------------------
CHRONO_DATA = {
    "D": [-1528, 17716, 19382],
    "s": [-131968728, 1530705600, 1674631932],
    "ms": [-131968727238, 1530705600000, 1674631932929],
    "us": [-131968727238000, 1530705600000000, 1674631932929000],
    "ns": [-131968727238000000, 1530705600000000000, 1674631932929000000],
}
_UNITS = ["D", "s", "ms", "us", "ns"]
for i, u in enumerate(_UNITS):
    for j in range(i, 5):  # DownCastingFloorsValues: every equal-or-finer chrono type to this one
        for src in (12 + j, 17 + j):
            for dst in (12 + i, 17 + i):
                _add(src="cast_tests.cpp:315 DownCastingFloorsValues", fn="cast", type=src, to=dst, values=CHRONO_DATA[_UNITS[j]],
                     expect=CHRONO_DATA[u], expect_type=dst)
# CastToTimestamps / CastFromTimestamps AllValid: duration X <-> timestamp X keeps the ticks
for i, u in enumerate(_UNITS):
    _add(src="cast_tests.cpp:362 CastToTimestamps", fn="cast", type=17 + i, to=12 + i, values=CHRONO_DATA[u], expect=CHRONO_DATA[u],
         expect_type=12 + i)
    _add(src="cast_tests.cpp:392 CastFromTimestamps", fn="cast", type=12 + i, to=17 + i, values=CHRONO_DATA[u],
         expect=CHRONO_DATA[u], expect_type=17 + i)
    _add(src="cast_tests.cpp:421 CastFromTimestamps WithNulls", fn="cast", type=12 + i, to=17 + i, values=CHRONO_DATA[u],
         valid=[True, False, True], expect=[CHRONO_DATA[u][0], None, CHRONO_DATA[u][2]], expect_type=17 + i)
# CastToDurations (integral types -> every duration: the tick counts) and CastFromDurations (durations -> numeric)
for t in [INT8, INT16, INT32, INT64, UINT8, UINT16, UINT32, UINT64, BOOL8]:
    _v = [1, 0, 1, 1] if t == BOOL8 else [1, 2, 3, 100]
    for d in range(17, 22):
        _add(src="cast_tests.cpp:455 CastToDurations", fn="cast", type=t, to=d, values=_v, expect=[int(x) for x in _v], expect_type=d)
for t in NUMERIC:
    for d in range(17, 22):
        _v = [1, 0, 1, 1] if t == BOOL8 else [1, 2, 3, 100]
        _add(src="cast_tests.cpp:487 CastFromDurations", fn="cast", type=d, to=t, values=_v,
             expect=[bool(x) for x in _v] if t == BOOL8 else _v, expect_type=t)
        _add(src="cast_tests.cpp:517 CastFromDurations WithNulls", fn="cast", type=d, to=t, values=_v,
             valid=[True, False, True, False], expect=[(bool(_v[0]) if t == BOOL8 else _v[0]), None,
                                                      (bool(_v[2]) if t == BOOL8 else _v[2]), None], expect_type=t)
# timestamps <-> numeric are not castable
for ts in range(12, 17):
    _add(src="cast_tests.cpp timestamp -> numeric", fn="cast", type=ts, to=INT64, values=[1, 2], raises="RuntimeError")
    _add(src="cast_tests.cpp numeric -> timestamp", fn="cast", type=INT64, to=ts, values=[1, 2], raises="RuntimeError")
# IsIdempotent: timestamp -> its duration -> the timestamp again ("to" lists the casts in order)
for i, u in enumerate(_UNITS):
    _add(src="cast_tests.cpp:206 IsIdempotent (timestamps)", fn="cast", type=12 + i, to=[17 + i, 12 + i], values=CHRONO_DATA[u],
         expect=CHRONO_DATA[u], expect_type=12 + i)
    _add(src="cast_tests.cpp:247 IsIdempotent (durations)", fn="cast", type=17 + i, to=[12 + i, 17 + i], values=CHRONO_DATA[u],
         expect=CHRONO_DATA[u], expect_type=17 + i)
