"""pylibcudf.binaryop twin (python/pylibcudf/pylibcudf/binaryop.pyx; cpp/include/cudf/binaryop.hpp) over b2_binary_operation /
_cs / _sc and b2_binary_is_supported_operation (cudf_b200/csrc/binaryop*.cu: one streaming kernel per call).

Fixed-width operands: INT8..UINT64, FLOAT32, FLOAT64 and BOOL8 in any combination; timestamps and durations only against the same
type, for comparisons and NULL_MAX / NULL_MIN. Semantics, undefined values and errors: include/cudf_b200.h."""
from __future__ import annotations

import ctypes as C
import enum

from .. import _lib
from .._lib import check, lib
from .column import Column, Scalar
from .types import DataType


class BinaryOperator(enum.IntEnum):  # cudf::binary_operator (cpp/include/cudf/binaryop.hpp:30-84): values are ABI
    ADD = 0
    SUB = 1
    MUL = 2
    DIV = 3
    TRUE_DIV = 4
    FLOOR_DIV = 5
    MOD = 6
    PMOD = 7
    PYMOD = 8
    POW = 9
    INT_POW = 10
    LOG_BASE = 11
    ATAN2 = 12
    SHIFT_LEFT = 13
    SHIFT_RIGHT = 14
    SHIFT_RIGHT_UNSIGNED = 15
    BITWISE_AND = 16
    BITWISE_OR = 17
    BITWISE_XOR = 18
    LOGICAL_AND = 19
    LOGICAL_OR = 20
    EQUAL = 21
    NOT_EQUAL = 22
    LESS = 23
    GREATER = 24
    LESS_EQUAL = 25
    GREATER_EQUAL = 26
    NULL_EQUALS = 27
    NULL_NOT_EQUALS = 28
    NULL_MAX = 29
    NULL_MIN = 30
    GENERIC_BINARY = 31
    NULL_LOGICAL_AND = 32
    NULL_LOGICAL_OR = 33
    INVALID_BINARY = 34


def binary_operation(lhs: Column | Scalar, rhs: Column | Scalar, op: BinaryOperator, output_type: DataType, stream=None,
                     mr=None) -> Column:
    """op(lhs[i], rhs[i]) as a column of `output_type`; a Scalar operand stands for every row. At least one operand is a Column."""
    out = C.c_void_p()
    s, o, t = _lib.stream_arg(stream), int(op), int(output_type.id())
    if isinstance(lhs, Column) and isinstance(rhs, Column):
        lv, rv = lhs._view(), rhs._view()
        check(lib.b2_binary_operation(C.byref(lv), C.byref(rv), o, t, s, C.byref(out)))
    elif isinstance(lhs, Column) and isinstance(rhs, Scalar):
        lv = lhs._view()
        check(lib.b2_binary_operation_cs(C.byref(lv), C.c_void_p(rhs._handle), o, t, s, C.byref(out)))
    elif isinstance(lhs, Scalar) and isinstance(rhs, Column):
        rv = rhs._view()
        check(lib.b2_binary_operation_sc(C.c_void_p(lhs._handle), C.byref(rv), o, t, s, C.byref(out)))
    else:
        raise ValueError("binary_operation: at least one operand must be a Column, and both a Column or a Scalar")
    return Column._from_handle(out.value)


def is_supported_operation(out: DataType, lhs: DataType, rhs: DataType, op: BinaryOperator) -> bool:
    """Whether binary_operation accepts these types for `op` (cudf::binops::is_supported_operation)."""
    r = C.c_int32(0)
    check(lib.b2_binary_is_supported_operation(int(out.id()), int(lhs.id()), int(rhs.id()), int(op), C.byref(r)))
    return bool(r.value)
