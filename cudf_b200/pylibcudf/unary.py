"""pylibcudf.unary twin (python/pylibcudf/pylibcudf/unary.pyx; cpp/include/cudf/unary.hpp) over b2_unary_operation, b2_cast,
b2_is_supported_cast, b2_is_null / b2_is_valid and b2_is_nan / b2_is_not_nan (cudf_b200/csrc/unary*.cu: one streaming kernel
per call).

Fixed-width columns only; decimal, dictionary, string and nested types are not held here. Semantics, undefined values and errors:
include/cudf_b200.h."""
from __future__ import annotations

import ctypes as C
import enum

import numpy as np

from .. import _lib
from .._lib import check, lib
from .column import Column
from .types import DataType, _NP


class UnaryOperator(enum.IntEnum):  # cudf::unary_operator (cpp/include/cudf/unary.hpp:32-57): values are ABI
    SIN = 0
    COS = 1
    TAN = 2
    ARCSIN = 3
    ARCCOS = 4
    ARCTAN = 5
    SINH = 6
    COSH = 7
    TANH = 8
    ARCSINH = 9
    ARCCOSH = 10
    ARCTANH = 11
    EXP = 12
    LOG = 13
    SQRT = 14
    CBRT = 15
    CEIL = 16
    FLOOR = 17
    ABS = 18
    RINT = 19
    BIT_COUNT = 20
    BIT_INVERT = 21
    NOT = 22
    NEGATE = 23


def _call(fn, input: Column, *args, stream=None) -> Column:
    out = C.c_void_p()
    v = input._view()
    check(fn(C.byref(v), *args, _lib.stream_arg(stream), C.byref(out)))
    return Column._from_handle(out.value)


def unary_operation(input: Column, op: UnaryOperator, stream=None, mr=None) -> Column:
    """op(input[i]); the output type is the input's, INT32 for BIT_COUNT and BOOL8 for NOT."""
    return _call(lib.b2_unary_operation, input, int(op), stream=stream)


def is_null(input: Column, stream=None, mr=None) -> Column:
    """A BOOL8 column without a mask: True where input is null."""
    return _call(lib.b2_is_null, input, stream=stream)


def is_valid(input: Column, stream=None, mr=None) -> Column:
    """A BOOL8 column without a mask: True where input is valid."""
    return _call(lib.b2_is_valid, input, stream=stream)


def cast(input: Column, data_type: DataType, stream=None, mr=None) -> Column:
    """input converted to `data_type` (static_cast for numbers, chrono::floor between time units)."""
    return _call(lib.b2_cast, input, int(data_type.id()), stream=stream)


def is_supported_cast(from_: DataType, to: DataType) -> bool:
    """Whether cast accepts this pair of types (cudf::is_supported_cast)."""
    r = C.c_int32(0)
    check(lib.b2_is_supported_cast(int(from_.id()), int(to.id()), C.byref(r)))
    return bool(r.value)


def _bit_castable(from_: DataType, to: DataType) -> bool:
    """cudf::is_bit_castable over the types held here: both fixed-width with the same storage width."""
    f, t = _NP.get(from_.id()), _NP.get(to.id())
    return f is not None and t is not None and np.dtype(f).itemsize == np.dtype(t).itemsize


def bit_cast(input: Column, data_type: DataType, stream=None, mr=None) -> Column:
    """A new column of `data_type` holding a copy of input's bits and mask (pylibcudf's bit_cast returns an owning column).
    Both types must be fixed-width with the same storage width; otherwise RuntimeError (cudf::logic_error)."""
    if not _bit_castable(input.type(), data_type):
        raise RuntimeError(f"bit_cast: {input.type().id()!r} and {data_type.id()!r} are not bit-castable")
    out = C.c_void_p()
    v = input._view()
    v.type_id = int(data_type.id())  # the same bits seen as the target type: a same-type cast is a copy
    check(lib.b2_cast(C.byref(v), int(data_type.id()), _lib.stream_arg(stream), C.byref(out)))
    return Column._from_handle(out.value)


def is_nan(input: Column, stream=None, mr=None) -> Column:
    """A BOOL8 column without a mask: True where a FLOAT32 / FLOAT64 input is NaN (a null row is False)."""
    return _call(lib.b2_is_nan, input, stream=stream)


def is_not_nan(input: Column, stream=None, mr=None) -> Column:
    """A BOOL8 column without a mask: True where a FLOAT32 / FLOAT64 input is not NaN (a null row is True)."""
    return _call(lib.b2_is_not_nan, input, stream=stream)


__all__ = ["UnaryOperator", "unary_operation", "is_null", "is_valid", "cast", "is_supported_cast", "bit_cast", "is_nan",
           "is_not_nan"]
