"""pylibcudf-named API of the H100 hot path (sorting, join, groupby, reduce, copying, aggregation, null_mask, stream_compaction,
binaryop, unary, replace)."""
from . import (aggregation, binaryop, contiguous_split, copying, groupby, interop, join, null_mask, partitioning, reduce, replace,
               sorting, stream_compaction, types, unary)
from .column import Column, DeviceSpan, Scalar, Table
from .types import (DataType, MaskState, NanEquality, NullEquality, NullOrder, NullPolicy, Order, OutOfBoundsPolicy, RankMethod,
                    Sorted, TypeId)

__all__ = [
    "aggregation", "binaryop", "contiguous_split", "copying", "groupby", "interop", "join", "null_mask", "partitioning", "reduce", "replace", "sorting",
    "stream_compaction", "types", "unary", "Column", "DeviceSpan", "Scalar", "Table", "DataType", "MaskState", "NanEquality", "NullEquality",
    "NullOrder", "NullPolicy", "Order", "OutOfBoundsPolicy", "RankMethod", "Sorted", "TypeId",
]
