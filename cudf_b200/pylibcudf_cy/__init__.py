"""Compiled (Cython) binding of the hot path: `cudf_b200.pylibcudf_cy` has the module layout of pylibcudf
(`Column`, `Table`, `binaryop`, `sorting`, `join`, `groupby`, `reduce`, `copying`, `partitioning`, `null_mask`, `contiguous_split`, `stream_compaction`, `unary`, `replace`, `aggregation`, `types`) with the operations implemented in
`_core.pyx` as typed, GIL-releasing calls into libcudf_b200.so (declared in libcudf_b200.pxd). Enumerations, DataType,
Aggregation and Scalar are the pure-Python classes of the ctypes twin `cudf_b200.pylibcudf`.

The extension is built in-tree by `cudf_b200.pylibcudf_cy.build_cy.build()` (called from `__graft_entry__.build()`); importing
this package without it raises ImportError — there is no fallback to the ctypes twin."""
from .. import _lib  # loads libcudf_b200.so first (the extension links against it)
from ..pylibcudf import aggregation, types
from ..pylibcudf.column import Scalar
from ..pylibcudf.types import (DataType, NanEquality, NullEquality, NullOrder, NullPolicy, Order, OutOfBoundsPolicy, Sorted, TypeId)
from . import _core
from ._core import Column, Table
from . import (binaryop, contiguous_split, copying, groupby, join, null_mask, partitioning, reduce, replace, sorting,
               stream_compaction, unary)

__all__ = ["Column", "Table", "Scalar", "DataType", "TypeId", "Order", "NullOrder", "NullPolicy", "NullEquality", "NanEquality", "Sorted",
           "OutOfBoundsPolicy", "aggregation", "types", "binaryop", "sorting", "join", "groupby", "reduce", "copying", "null_mask", "partitioning", "contiguous_split",
           "stream_compaction", "unary", "replace"]
