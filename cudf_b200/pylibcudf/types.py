"""Type tags and enums — values are ABI (cpp/include/cudf/types.hpp:76-77,99-216; python/pylibcudf/pylibcudf/types.pyx)."""
from __future__ import annotations

import enum

import numpy as np

size_type = np.int32
bitmask_type = np.uint32


class TypeId(enum.IntEnum):
    EMPTY = 0
    INT8 = 1
    INT16 = 2
    INT32 = 3
    INT64 = 4
    UINT8 = 5
    UINT16 = 6
    UINT32 = 7
    UINT64 = 8
    FLOAT32 = 9
    FLOAT64 = 10
    BOOL8 = 11
    TIMESTAMP_DAYS = 12
    TIMESTAMP_SECONDS = 13
    TIMESTAMP_MILLISECONDS = 14
    TIMESTAMP_MICROSECONDS = 15
    TIMESTAMP_NANOSECONDS = 16
    DURATION_DAYS = 17
    DURATION_SECONDS = 18
    DURATION_MILLISECONDS = 19
    DURATION_MICROSECONDS = 20
    DURATION_NANOSECONDS = 21
    # not fixed-width: no column of these types exists here; operations reject them
    DICTIONARY32 = 22
    STRING = 23
    LIST = 24
    DECIMAL32 = 25
    DECIMAL64 = 26
    DECIMAL128 = 27
    STRUCT = 28
    NUM_TYPE_IDS = 29


class Order(enum.IntEnum):
    ASCENDING = 0
    DESCENDING = 1


class NullOrder(enum.IntEnum):
    AFTER = 0
    BEFORE = 1


class NullPolicy(enum.IntEnum):
    EXCLUDE = 0
    INCLUDE = 1


class RankMethod(enum.IntEnum):  # cudf::rank_method (cpp/include/cudf/aggregation.hpp:37-43)
    FIRST = 0
    AVERAGE = 1
    MIN = 2
    MAX = 3
    DENSE = 4


class NullEquality(enum.IntEnum):
    EQUAL = 0
    UNEQUAL = 1


class NanEquality(enum.IntEnum):  # cudf::nan_equality (types.hpp)
    ALL_EQUAL = 0
    UNEQUAL = 1


class Sorted(enum.IntEnum):
    NO = 0
    YES = 1


class MaskState(enum.IntEnum):
    UNALLOCATED = 0
    UNINITIALIZED = 1
    ALL_VALID = 2
    ALL_NULL = 3


class OutOfBoundsPolicy(enum.IntEnum):
    NULLIFY = 0
    DONT_CHECK = 1


_NP = {
    TypeId.INT8: np.int8, TypeId.INT16: np.int16, TypeId.INT32: np.int32, TypeId.INT64: np.int64,
    TypeId.UINT8: np.uint8, TypeId.UINT16: np.uint16, TypeId.UINT32: np.uint32, TypeId.UINT64: np.uint64,
    TypeId.FLOAT32: np.float32, TypeId.FLOAT64: np.float64, TypeId.BOOL8: np.bool_,
    TypeId.TIMESTAMP_DAYS: np.int32, TypeId.DURATION_DAYS: np.int32,
}
for _t in (TypeId.TIMESTAMP_SECONDS, TypeId.TIMESTAMP_MILLISECONDS, TypeId.TIMESTAMP_MICROSECONDS,
           TypeId.TIMESTAMP_NANOSECONDS, TypeId.DURATION_SECONDS, TypeId.DURATION_MILLISECONDS,
           TypeId.DURATION_MICROSECONDS, TypeId.DURATION_NANOSECONDS):
    _NP[_t] = np.int64


class DataType:
    """cudf::data_type (types.hpp:278-340) for fixed-width, scale-free types."""

    __slots__ = ("_id",)

    def __init__(self, type_id: TypeId):
        self._id = TypeId(type_id)

    def id(self) -> TypeId:
        return self._id

    def numpy_dtype(self) -> np.dtype:
        return np.dtype(_NP[self._id])

    @property
    def itemsize(self) -> int:
        return self.numpy_dtype().itemsize

    @staticmethod
    def from_numpy(dtype) -> "DataType":
        dtype = np.dtype(dtype)
        if dtype.kind == "M" or dtype.kind == "m":
            unit = np.datetime_data(dtype)[0]
            base = {"D": 0, "s": 1, "ms": 2, "us": 3, "ns": 4}[unit]
            return DataType(TypeId((12 if dtype.kind == "M" else 17) + base))
        for tid in (TypeId.INT8, TypeId.INT16, TypeId.INT32, TypeId.INT64, TypeId.UINT8, TypeId.UINT16,
                    TypeId.UINT32, TypeId.UINT64, TypeId.FLOAT32, TypeId.FLOAT64, TypeId.BOOL8):
            if np.dtype(_NP[tid]) == dtype:
                return DataType(tid)
        raise TypeError(f"unsupported dtype {dtype}")

    def __eq__(self, other):
        return isinstance(other, DataType) and other._id == self._id

    def __hash__(self):
        return hash(self._id)

    def __repr__(self):
        return f"DataType({self._id.name})"
