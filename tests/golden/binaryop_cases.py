"""Known answers for cudf::binary_operation, transcribed from the reference tree (file:line in "src"):
cpp/tests/binaryop/binop-compiled-test.cpp, binop-null-test.cpp and binop-verify-input-test.cpp.

Each case: "op" (cudf::binary_operator value), "lhs" / "rhs" = (values with None for null, dtype) for a column or
{"scalar": value or None, "dtype": dtype} for a scalar, "out" (dtype name), and either "expect" (values with None for null) or
"raises" (the Python exception class name: ValueError = std::invalid_argument, RuntimeError = cudf::logic_error). The rule tables
of the null-aware operators are the operators' definitions in cpp/src/binaryop/compiled/operation.cuh, which the compiled test
checks on random columns; here they are written out over every (valid, null) pairing."""

I64_MAX, I64_MIN = 2**63 - 1, -(2**63)
N = None

CASES = [
    # IntPow_SpecialCases: values that a round trip through double gets wrong
    {"src": "binop-compiled-test.cpp:390-407 (int32)", "op": 10, "lhs": ([3, -3, 8, -8], "int32"), "rhs": ([1, 1, 7, 7], "int32"),
     "out": "int32", "expect": [3, -3, 2097152, -2097152]},
    {"src": "binop-compiled-test.cpp:390-407 (int64)", "op": 10, "lhs": ([3, -3, 8, -8], "int64"), "rhs": ([1, 1, 7, 7], "int64"),
     "out": "int64", "expect": [3, -3, 2097152, -2097152]},
    # FloorDivInt64Positive / RoundNegativeInf: exact at the int64 limits, rounding toward -inf
    {"src": "binop-compiled-test.cpp:409-430", "op": 5, "lhs": ([I64_MAX, I64_MAX - 10, I64_MAX - 100], "int64"),
     "rhs": ([10, 10, 10], "int64"), "out": "int64", "expect": [I64_MAX // 10, (I64_MAX - 10) // 10, (I64_MAX - 100) // 10]},
    {"src": "binop-compiled-test.cpp:432-453", "op": 5, "lhs": ([I64_MIN, I64_MIN + 10, I64_MIN + 100], "int64"),
     "rhs": ([10, 10, 10], "int64"), "out": "int64",
     "expect": [-922337203685477581, -922337203685477580, -922337203685477571]},
    # NullEquals / NullNotEquals (int16, int8 -> bool): null == null is true, null == value false, every row valid
    {"src": "binop-compiled-test.cpp:676-690", "op": 27, "lhs": ([1, 1, N, N, 5], "int16"), "rhs": ([1, N, 1, N, 6], "int8"),
     "out": "bool", "expect": [True, False, False, True, False]},
    {"src": "binop-compiled-test.cpp:710-724", "op": 28, "lhs": ([1, 1, N, N, 5], "int16"), "rhs": ([1, N, 1, N, 6], "int8"),
     "out": "bool", "expect": [False, True, True, False, True]},
    # NullMax / NullMin (uint16, uint32 -> uint16; double, uint64 -> double): the valid operand, null when both are
    {"src": "binop-compiled-test.cpp:744-758", "op": 29, "lhs": ([3, 3, N, N], "uint16"), "rhs": ([7, N, 7, N], "uint32"),
     "out": "uint16", "expect": [7, 3, 7, N]},
    {"src": "binop-compiled-test.cpp:760-774", "op": 30, "lhs": ([3.5, 3.5, N, N], "float64"), "rhs": ([7, N, 7, N], "uint64"),
     "out": "float64", "expect": [3.5, 3.5, 7.0, N]},
    # NullLogicalAnd / NullLogicalOr: (null, false) is false, (null, true) is true, otherwise null when an operand is
    {"src": "binop-compiled-test.cpp:564-580", "op": 32, "lhs": ([True, True, False, N, N, N, True, False], "bool"),
     "rhs": ([N, True, N, False, True, N, False, False], "bool"), "out": "bool",
     "expect": [N, True, False, False, N, N, False, False]},
    {"src": "binop-compiled-test.cpp:582-596", "op": 33, "lhs": ([True, True, False, N, N, N, True, False], "bool"),
     "rhs": ([N, True, N, False, True, N, False, False], "bool"), "out": "bool",
     "expect": [True, True, N, N, True, N, True, False]},
    # binop-null-test.cpp: a null scalar nulls every row; otherwise the AND of the validities
    {"src": "binop-null-test.cpp:32-45", "op": 0, "lhs": {"scalar": None, "dtype": "int32"}, "rhs": (list(range(10)), "int32"),
     "out": "int32", "expect": [N] * 10},
    {"src": "binop-null-test.cpp:47-57", "op": 0, "lhs": {"scalar": 1, "dtype": "int32"}, "rhs": (list(range(10)), "int32"),
     "out": "int32", "expect": list(range(1, 11))},
    {"src": "binop-null-test.cpp:59-71", "op": 0, "lhs": {"scalar": None, "dtype": "int32"}, "rhs": (list(range(10)), "int32"),
     "out": "int32", "expect": [N] * 10},
    {"src": "binop-null-test.cpp:73-83", "op": 0, "lhs": {"scalar": 1, "dtype": "int32"}, "rhs": ([N] * 10, "int32"),
     "out": "int32", "expect": [N] * 10},
    {"src": "binop-null-test.cpp:85-96", "op": 0, "lhs": ([N] * 10, "int32"), "rhs": (list(range(10)), "int32"),
     "out": "int32", "expect": [N] * 10},
    {"src": "binop-null-test.cpp:110-122", "op": 0, "lhs": (list(range(9, -1, -1)), "int32"), "rhs": (list(range(10)), "int32"),
     "out": "int32", "expect": [9] * 10},
    # binop-verify-input-test.cpp: an output type id outside cudf::type_id is a logic_error; differing column sizes
    # std::invalid_argument
    {"src": "binop-verify-input-test.cpp:13-22", "op": 0, "lhs": {"scalar": 1, "dtype": "int64"},
     "rhs": (list(range(10)), "int64"), "out": 29, "raises": "RuntimeError"},
    {"src": "binop-verify-input-test.cpp:24-32", "op": 0, "lhs": ([1], "int64"), "rhs": (list(range(10)), "int64"), "out": "int64",
     "raises": "ValueError"},
]

# (op, out, lhs, rhs, supported) spot rows of util.cpp's rule (cudf type ids): bitwise operators and shifts are not defined on
# floats, SHIFT_RIGHT_UNSIGNED not on bool, comparisons only write BOOL8, arithmetic writes any numeric type.
SUPPORTED_SPOTS = [
    (16, 9, 9, 9, False), (16, 3, 3, 9, False), (16, 10, 3, 3, True), (13, 4, 4, 10, False), (15, 11, 11, 11, False),
    (15, 3, 11, 1, True), (10, 4, 4, 9, False), (10, 11, 11, 11, True), (24, 3, 4, 9, False), (24, 11, 4, 9, True),
    (0, 11, 9, 1, True), (9, 1, 11, 11, True), (31, 4, 4, 4, False), (19, 11, 9, 10, True), (29, 4, 12, 12, False),
    (29, 12, 12, 12, True), (21, 11, 12, 13, False), (0, 4, 12, 12, False), (0, 23, 4, 4, False),
]
