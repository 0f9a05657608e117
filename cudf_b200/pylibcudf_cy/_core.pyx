# cython: language_level=3, boundscheck=False, wraparound=False
"""Compiled (Cython) binding of the hot path over the C ABI — the layer python/pylibcudf/pylibcudf/*.pyx is for libcudf:
`cdef class Column / Table` own the `b2_column` handles the library returns, every operation is a typed `nogil` call into
`libcudf_b200.so` declared in libcudf_b200.pxd (checked by the C compiler against include/cudf_b200.h), errors surface as the
exception classes of python/pylibcudf/pylibcudf/exception_handler.pxd:29-66.

Reference counterparts: column.pyx / table.pyx (Column, Table), sorting.pyx:37-79,333-520, join.pyx:63-205,
groupby.pyx:36-243, reduce.pyx:48-157, copying.pyx:64-113. Enumerations, DataType, Aggregation and Scalar are shared with the
ctypes twin (`cudf_b200.pylibcudf`); `Column.to_plc()` / `Column.from_plc()` convert between the two Column classes without
copying, which is also how host <-> device transfers (`from_numpy`, `to_numpy`, `from_torch`, `to_torch`) are provided.
"""
from libc.stdint cimport int32_t, int64_t, uint8_t, uint32_t, uint64_t, uintptr_t
from libc.stdlib cimport calloc, free

from cudf_b200.pylibcudf_cy.libcudf_b200 cimport *

from cudf_b200.pylibcudf import column as _plc_column
from cudf_b200.pylibcudf.column import DeviceSpan
from cudf_b200.pylibcudf.column import Scalar as _PlcScalar
from cudf_b200.pylibcudf.types import DataType, NullPolicy, Sorted, TypeId

_STATUS_EXC = {
    1: RuntimeError,   # cudf::logic_error
    2: ValueError,     # std::invalid_argument
    3: TypeError,      # cudf::data_type_error
    4: IndexError,     # std::out_of_range
    5: MemoryError,    # std::bad_alloc
    6: RuntimeError,   # cudf::cuda_error
}


cdef int check(b2_status st) except -1:
    if st != 0:
        msg = b2_last_error().decode("utf-8", "replace")
        raise _STATUS_EXC.get(<int>st, RuntimeError)(msg)
    return 0


cdef b2_stream _stream(object stream) except? NULL:
    """None = the current stream of the ctypes twin's rule (torch's current stream on a GPU); an int / object with
    `.cuda_stream` / `.ptr` otherwise."""
    from cudf_b200 import _lib

    cdef object s = _lib.stream_arg(stream)  # ctypes c_void_p
    return <b2_stream><uintptr_t>(s.value or 0)


def version():
    return b2_version().decode()


def kernel_launch_count():
    return int(b2_kernel_launch_count())


# ---------------------------------------------------------------------------------------------------------------------
# Column / Table
# ---------------------------------------------------------------------------------------------------------------------
cdef class Column:
    """Non-owning view fields (cudf::column_view) + what keeps the memory alive: a `b2_column` handle returned by the
    library (freed with the object) or arbitrary Python owners (tensors, other columns)."""
    cdef b2_column_view v
    cdef b2_column* handle
    cdef object owners

    def __cinit__(self):
        self.handle = NULL
        self.owners = None
        self.v.type_id = 0
        self.v.size = 0
        self.v.data = NULL
        self.v.null_mask = NULL
        self.v.null_count = 0
        self.v.offset = 0

    def __dealloc__(self):
        if self.handle != NULL:
            b2_column_free(self.handle)
            self.handle = NULL

    @staticmethod
    cdef Column from_handle(b2_column* h):
        cdef Column c = Column.__new__(Column)
        c.handle = h
        check(b2_column_view_of(h, &c.v))
        return c

    @staticmethod
    def from_pointers(data_type, Py_ssize_t size, uintptr_t data_ptr, uintptr_t mask_ptr=0, int null_count=0, int offset=0, owners=None):
        """A view of device memory somebody else owns (`owners` is kept alive as long as the column)."""
        cdef Column c = Column.__new__(Column)
        c.v.type_id = int(data_type.id())
        c.v.size = <int32_t>size
        c.v.data = <const void*>data_ptr
        c.v.null_mask = <const uint32_t*>mask_ptr
        c.v.null_count = null_count
        c.v.offset = offset
        c.owners = owners
        return c

    @staticmethod
    def from_cuda_array_interface(obj, mask=None, null_count=None, int offset=0, size=None):
        """Zero-copy from anything exposing `__cuda_array_interface__` (torch / cupy / numba device arrays); `mask` is a device
        array of Arrow validity words."""
        import numpy as np

        iface = obj.__cuda_array_interface__
        if len(iface["shape"]) != 1 or iface.get("strides") not in (None, (np.dtype(iface["typestr"]).itemsize,)):
            raise ValueError("a contiguous 1-D device array is required")
        dt = DataType.from_numpy(np.dtype(iface["typestr"]))
        cdef Py_ssize_t n = iface["shape"][0] - offset if size is None else size
        cdef uintptr_t mptr = 0
        cdef int32_t nulls = 0
        if mask is not None:
            mptr = mask.__cuda_array_interface__["data"][0]
            if null_count is None:
                check(b2_null_count(<const uint32_t*>mptr, offset, offset + <int32_t>n, _stream(None), &nulls))
            else:
                nulls = null_count
        return Column.from_pointers(dt, n, iface["data"][0], mptr, nulls, offset, [obj, mask])

    @staticmethod
    def from_plc(col):
        """Shares the memory of a `cudf_b200.pylibcudf.Column` (the ctypes twin)."""
        return Column.from_pointers(col._type, col._size, col._data, col._mask, col._null_count, col._offset, [col])

    def to_plc(self):
        return _plc_column.Column(DataType(TypeId(self.v.type_id)), self.v.size, <uintptr_t>self.v.data, <uintptr_t>self.v.null_mask,
                                  self.v.null_count, self.v.offset, [self])

    # host <-> device transfers and torch interop go through the ctypes twin's helpers (plumbing, not the product)
    @staticmethod
    def from_numpy(values, valid=None, dtype=None, **kw):
        return Column.from_plc(_plc_column.Column.from_numpy(values, valid, dtype, **kw))

    @staticmethod
    def from_torch(data, mask=None, null_count=None, dtype=None, int offset=0, size=None):
        return Column.from_plc(_plc_column.Column.from_torch(data, mask, null_count, dtype, offset, size))

    def to_numpy(self):
        return self.to_plc().to_numpy()

    def to_torch(self):
        return self.to_plc().to_torch()

    # ---- accessors (names follow pylibcudf.Column) ----
    def type(self):
        return DataType(TypeId(self.v.type_id))

    def size(self):
        return self.v.size

    def null_count(self):
        return self.v.null_count

    def offset(self):
        return self.v.offset

    def nullable(self):
        return self.v.null_mask != NULL

    def has_nulls(self):
        return self.v.null_count > 0

    def data(self):
        dt = DataType(TypeId(self.v.type_id)).numpy_dtype()
        return DeviceSpan(<uintptr_t>self.v.data + self.v.offset * dt.itemsize, self.v.size, dt, self)

    def null_mask(self):
        import numpy as np

        if self.v.null_mask == NULL:
            return None
        return DeviceSpan(<uintptr_t>self.v.null_mask, (self.v.offset + self.v.size + 31) // 32, np.uint32, self)

    def slice(self, int begin, int end):
        """cudf::slice of one range: shares memory, moves `offset`."""
        if not (0 <= begin <= end <= self.v.size):
            raise IndexError("slice out of range")
        cdef int32_t nulls = 0
        if self.v.null_mask != NULL and self.v.null_count:
            check(b2_null_count(self.v.null_mask, self.v.offset + begin, self.v.offset + end, _stream(None), &nulls))
        return Column.from_pointers(self.type(), end - begin, <uintptr_t>self.v.data, <uintptr_t>self.v.null_mask, nulls,
                                    self.v.offset + begin, [self])

    def __repr__(self):
        return f"Column({self.type()!r}, size={self.v.size}, null_count={self.v.null_count}, offset={self.v.offset})"


cdef class Table:
    cdef list cols

    def __init__(self, columns):
        self.cols = list(columns)
        cdef Column c
        if self.cols:
            n = (<Column>self.cols[0]).v.size
            for c in self.cols:
                if c.v.size != n:
                    raise ValueError("Column size mismatch")

    @staticmethod
    cdef Table from_handle(b2_table* t):
        cdef int32_t n = b2_table_num_columns(t)
        cdef int32_t cap = n if n > 0 else 1
        cdef b2_column** arr = <b2_column**>calloc(cap, sizeof(b2_column*))
        if arr == NULL:
            b2_table_free(t)
            raise MemoryError()
        cdef list out = []
        cdef int i
        try:
            check(b2_table_release(t, arr, cap))
            for i in range(n):
                out.append(Column.from_handle(arr[i]))
                arr[i] = NULL
        finally:
            for i in range(n):
                if arr[i] != NULL:
                    b2_column_free(arr[i])
            free(arr)
            b2_table_free(t)
        return Table(out)

    def columns(self):
        return list(self.cols)

    def num_columns(self):
        return len(self.cols)

    def num_rows(self):
        return (<Column>self.cols[0]).v.size if self.cols else 0


cdef class _TableView:
    """b2_table_view of a Table for the duration of one call (the column_view array lives here)."""
    cdef b2_column_view* arr
    cdef b2_table_view tv
    cdef object keep

    def __cinit__(self):
        self.arr = NULL

    def __dealloc__(self):
        if self.arr != NULL:
            free(self.arr)
            self.arr = NULL

    @staticmethod
    cdef _TableView of(Table t):
        cdef _TableView r = _TableView.__new__(_TableView)
        cdef Py_ssize_t n = len(t.cols)
        r.arr = <b2_column_view*>calloc(n if n > 0 else 1, sizeof(b2_column_view))
        if r.arr == NULL:
            raise MemoryError()
        cdef Py_ssize_t i
        for i in range(n):
            r.arr[i] = (<Column>t.cols[i]).v
        r.tv.columns = r.arr
        r.tv.num_columns = <int32_t>n
        r.keep = t
        return r


cdef class _Flags:
    """uint8 array of order / null-precedence flags (empty = the library's defaults)."""
    cdef uint8_t* p
    cdef int32_t n

    def __cinit__(self):
        self.p = NULL
        self.n = 0

    def __dealloc__(self):
        if self.p != NULL:
            free(self.p)
            self.p = NULL

    @staticmethod
    cdef _Flags of(object seq):
        cdef _Flags f = _Flags.__new__(_Flags)
        cdef list vals = [int(x) for x in (seq or [])]
        f.n = <int32_t>len(vals)
        f.p = <uint8_t*>calloc(f.n if f.n > 0 else 1, 1)
        if f.p == NULL:
            raise MemoryError()
        cdef int i
        for i in range(f.n):
            f.p[i] = <uint8_t>vals[i]
        return f


# ---------------------------------------------------------------------------------------------------------------------
# sorting (python/pylibcudf/pylibcudf/sorting.pyx:37-79,333-520)
# ---------------------------------------------------------------------------------------------------------------------
cdef Column _sorted_order(Table source_table, object column_order, object null_precedence, int stable, object stream):
    cdef _TableView tv = _TableView.of(source_table)
    cdef _Flags o = _Flags.of(column_order), p = _Flags.of(null_precedence)
    cdef b2_stream s = _stream(stream)
    cdef b2_column* out = NULL
    cdef b2_status st
    with nogil:
        st = b2_sorted_order(&tv.tv, o.p, o.n, p.p, p.n, stable, s, &out)
    check(st)
    return Column.from_handle(out)


cdef Table _sort(Table source_table, object column_order, object null_precedence, int stable, object stream):
    cdef _TableView tv = _TableView.of(source_table)
    cdef _Flags o = _Flags.of(column_order), p = _Flags.of(null_precedence)
    cdef b2_stream s = _stream(stream)
    cdef b2_table* out = NULL
    cdef b2_status st
    with nogil:
        st = b2_sort(&tv.tv, o.p, o.n, p.p, p.n, stable, s, &out)
    check(st)
    return Table.from_handle(out)


cdef Table _sort_by_key(Table values, Table keys, object column_order, object null_precedence, int stable, object stream):
    cdef _TableView vv = _TableView.of(values), kv = _TableView.of(keys)
    cdef _Flags o = _Flags.of(column_order), p = _Flags.of(null_precedence)
    cdef b2_stream s = _stream(stream)
    cdef b2_table* out = NULL
    cdef b2_status st
    with nogil:
        st = b2_sort_by_key(&vv.tv, &kv.tv, o.p, o.n, p.p, p.n, stable, s, &out)
    check(st)
    return Table.from_handle(out)


def sorted_order(Table source_table, column_order, null_precedence, stream=None, mr=None):
    return _sorted_order(source_table, column_order, null_precedence, 0, stream)


def stable_sorted_order(Table source_table, column_order, null_precedence, stream=None, mr=None):
    return _sorted_order(source_table, column_order, null_precedence, 1, stream)


def sort(Table source_table, column_order, null_precedence, stream=None, mr=None):
    return _sort(source_table, column_order, null_precedence, 0, stream)


def stable_sort(Table source_table, column_order, null_precedence, stream=None, mr=None):
    return _sort(source_table, column_order, null_precedence, 1, stream)


def sort_by_key(Table values, Table keys, column_order, null_precedence, stream=None, mr=None):
    return _sort_by_key(values, keys, column_order, null_precedence, 0, stream)


def stable_sort_by_key(Table values, Table keys, column_order, null_precedence, stream=None, mr=None):
    return _sort_by_key(values, keys, column_order, null_precedence, 1, stream)


# ---------------------------------------------------------------------------------------------------------------------
# copying.gather (python/pylibcudf/pylibcudf/copying.pyx:64-113)
# ---------------------------------------------------------------------------------------------------------------------
def gather(Table source_table, Column gather_map, bounds_policy, stream=None, mr=None):
    cdef _TableView tv = _TableView.of(source_table)
    cdef int32_t pol = int(bounds_policy)
    cdef b2_stream s = _stream(stream)
    cdef b2_table* out = NULL
    cdef b2_status st
    with nogil:
        st = b2_gather(&tv.tv, &gather_map.v, pol, s, &out)
    check(st)
    return Table.from_handle(out)


# ---------------------------------------------------------------------------------------------------------------------
# stream compaction (python/pylibcudf/pylibcudf/stream_compaction.pyx; cpp/include/cudf/stream_compaction.hpp)
# ---------------------------------------------------------------------------------------------------------------------
cdef class _KeyIndices:
    """A C array of int32 key column indices (valid while the object lives)."""
    cdef int32_t* p
    cdef int32_t n

    def __cinit__(self, keys):
        keys = [int(k) for k in keys]
        self.n = len(keys)
        self.p = <int32_t*>calloc(max(self.n, 1), sizeof(int32_t))
        if self.p == NULL:
            raise MemoryError()
        for j in range(self.n):
            self.p[j] = keys[j]

    def __dealloc__(self):
        free(self.p)


cdef Table _mask_call(Table input, Column mask, int32_t deletion, stream):
    cdef _TableView tv = _TableView.of(input)
    cdef b2_stream s = _stream(stream)
    cdef b2_table* out = NULL
    cdef b2_status st
    with nogil:
        st = b2_apply_boolean_mask(&tv.tv, &mask.v, deletion, s, &out)
    check(st)
    return Table.from_handle(out)


def apply_boolean_mask(Table source_table, Column boolean_mask, stream=None, mr=None):
    """Rows where `boolean_mask` (BOOL8) is valid and true, in input order."""
    return _mask_call(source_table, boolean_mask, 0, stream)


def apply_deletion_mask(Table input, Column deletion_mask, stream=None, mr=None):  # noqa: A002
    """Rows where `deletion_mask` (BOOL8) is valid and false, in input order."""
    return _mask_call(input, deletion_mask, 1, stream)


cdef Table _threshold_call(Table input, keys, keep_threshold, bint nans, stream):
    cdef _TableView tv = _TableView.of(input)
    cdef _KeyIndices k = _KeyIndices(keys)
    cdef int32_t thr = k.n if keep_threshold is None else int(keep_threshold)
    cdef b2_stream s = _stream(stream)
    cdef b2_table* out = NULL
    cdef b2_status st
    with nogil:
        if nans:
            st = b2_drop_nans(&tv.tv, k.p, k.n, thr, s, &out)
        else:
            st = b2_drop_nulls(&tv.tv, k.p, k.n, thr, s, &out)
    check(st)
    return Table.from_handle(out)


def drop_nulls(Table source_table, keys, keep_threshold=None, stream=None, mr=None):
    """Rows with at least `keep_threshold` (default: all) valid columns among `keys`."""
    return _threshold_call(source_table, keys, keep_threshold, False, stream)


def drop_nans(Table source_table, keys, keep_threshold=None, stream=None, mr=None):
    """Rows with at least `keep_threshold` (default: all) non-NaN columns among the float `keys`; a null is not NaN."""
    return _threshold_call(source_table, keys, keep_threshold, True, stream)


def unique(Table input, keys, keep, nulls_equal, stream=None, mr=None):  # noqa: A002
    """Drops consecutive duplicate rows of the `keys` columns."""
    cdef _TableView tv = _TableView.of(input)
    cdef _KeyIndices k = _KeyIndices(keys)
    cdef int32_t kp = int(keep), ne = int(nulls_equal)
    cdef b2_stream s = _stream(stream)
    cdef b2_table* out = NULL
    cdef b2_status st
    with nogil:
        st = b2_unique(&tv.tv, k.p, k.n, kp, ne, s, &out)
    check(st)
    return Table.from_handle(out)


cdef Table _distinct_call(Table input, keys, keep, nulls_equal, nans_equal, int32_t stable, stream):
    cdef _TableView tv = _TableView.of(input)
    cdef _KeyIndices k = _KeyIndices(keys)
    cdef int32_t kp = int(keep), ne = int(nulls_equal), nn = int(nans_equal)
    cdef b2_stream s = _stream(stream)
    cdef b2_table* out = NULL
    cdef b2_status st
    with nogil:
        st = b2_distinct(&tv.tv, k.p, k.n, kp, ne, nn, stable, s, &out)
    check(st)
    return Table.from_handle(out)


def distinct(Table input, keys, keep, nulls_equal, nans_equal, stream=None, mr=None):  # noqa: A002
    """One row per set of equal `keys` rows; the order is unspecified (here: input order)."""
    return _distinct_call(input, keys, keep, nulls_equal, nans_equal, 0, stream)


def stable_distinct(Table input, keys, keep, nulls_equal, nans_equal, stream=None, mr=None):  # noqa: A002
    """The rows of `distinct`, in input order."""
    return _distinct_call(input, keys, keep, nulls_equal, nans_equal, 1, stream)


def distinct_indices(Table input, keep, nulls_equal, nans_equal, stream=None, mr=None):  # noqa: A002
    """INT32 indices of the rows `distinct` keeps over all columns of `input`, ascending."""
    cdef _TableView tv = _TableView.of(input)
    cdef int32_t kp = int(keep), ne = int(nulls_equal), nn = int(nans_equal)
    cdef b2_stream s = _stream(stream)
    cdef b2_column* out = NULL
    cdef b2_status st
    with nogil:
        st = b2_distinct_indices(&tv.tv, kp, ne, nn, s, &out)
    check(st)
    return Column.from_handle(out)


# ---------------------------------------------------------------------------------------------------------------------
# binary operations (python/pylibcudf/pylibcudf/binaryop.pyx; cpp/include/cudf/binaryop.hpp)
# ---------------------------------------------------------------------------------------------------------------------
def binary_operation(lhs, rhs, op, output_type, stream=None, mr=None):
    """op(lhs[i], rhs[i]) as a Column of `output_type`; each operand a Column or a Scalar, at least one a Column."""
    cdef int32_t o = int(op)
    cdef int32_t t = int(output_type.id())
    cdef b2_stream s = _stream(stream)
    cdef b2_column* out = NULL
    cdef b2_status st
    cdef Column lc
    cdef Column rc
    cdef const b2_scalar* sc
    if isinstance(lhs, Column) and isinstance(rhs, Column):
        lc, rc = lhs, rhs
        with nogil:
            st = b2_binary_operation(&lc.v, &rc.v, o, t, s, &out)
    elif isinstance(lhs, Column) and isinstance(rhs, _PlcScalar):
        lc = lhs
        sc = <const b2_scalar*><uintptr_t>rhs._handle
        with nogil:
            st = b2_binary_operation_cs(&lc.v, sc, o, t, s, &out)
    elif isinstance(lhs, _PlcScalar) and isinstance(rhs, Column):
        rc = rhs
        sc = <const b2_scalar*><uintptr_t>lhs._handle
        with nogil:
            st = b2_binary_operation_sc(sc, &rc.v, o, t, s, &out)
    else:
        raise ValueError("binary_operation: at least one operand must be a Column, and both a Column or a Scalar")
    check(st)
    return Column.from_handle(out)


def is_supported_operation(out, lhs, rhs, op):
    """Whether binary_operation accepts these types for `op` (cudf::binops::is_supported_operation)."""
    cdef int32_t r = 0
    check(b2_binary_is_supported_operation(int(out.id()), int(lhs.id()), int(rhs.id()), int(op), &r))
    return r != 0


# ---------------------------------------------------------------------------------------------------------------------
# unary operations and casts (python/pylibcudf/pylibcudf/unary.pyx; cpp/include/cudf/unary.hpp)
# ---------------------------------------------------------------------------------------------------------------------
def unary_operation(Column input, op, stream=None, mr=None):
    """op(input[i]); the output type is the input's, INT32 for BIT_COUNT and BOOL8 for NOT."""
    cdef int32_t o = int(op)
    cdef b2_stream s = _stream(stream)
    cdef b2_column* out = NULL
    cdef b2_status st
    with nogil:
        st = b2_unary_operation(&input.v, o, s, &out)
    check(st)
    return Column.from_handle(out)


def cast(Column input, data_type, stream=None, mr=None):
    """input converted to `data_type` (static_cast for numbers, chrono::floor between time units)."""
    cdef int32_t t = int(data_type.id())
    cdef b2_stream s = _stream(stream)
    cdef b2_column* out = NULL
    cdef b2_status st
    with nogil:
        st = b2_cast(&input.v, t, s, &out)
    check(st)
    return Column.from_handle(out)


def is_supported_cast(from_, to):
    """Whether cast accepts this pair of types (cudf::is_supported_cast)."""
    cdef int32_t r = 0
    check(b2_is_supported_cast(int(from_.id()), int(to.id()), &r))
    return r != 0


def bit_cast(Column input, data_type, stream=None, mr=None):
    """A new column of `data_type` holding a copy of input's bits and mask; both types fixed-width of the same storage width,
    otherwise RuntimeError (cudf::logic_error)."""
    from cudf_b200.pylibcudf.unary import _bit_castable
    if not _bit_castable(input.type(), data_type):
        raise RuntimeError(f"bit_cast: {input.type().id()!r} and {data_type.id()!r} are not bit-castable")
    cdef b2_column_view v = input.v
    v.type_id = int(data_type.id())  # the same bits seen as the target type: a same-type cast is a copy
    cdef b2_stream s = _stream(stream)
    cdef b2_column* out = NULL
    cdef b2_status st
    with nogil:
        st = b2_cast(&v, v.type_id, s, &out)
    check(st)
    return Column.from_handle(out)


def _predicate(Column input, int which, stream):
    cdef b2_stream s = _stream(stream)
    cdef b2_column* out = NULL
    cdef b2_status st
    with nogil:
        if which == 0:
            st = b2_is_null(&input.v, s, &out)
        elif which == 1:
            st = b2_is_valid(&input.v, s, &out)
        elif which == 2:
            st = b2_is_nan(&input.v, s, &out)
        else:
            st = b2_is_not_nan(&input.v, s, &out)
    check(st)
    return Column.from_handle(out)


def is_null(Column input, stream=None, mr=None):
    """A BOOL8 column without a mask: True where input is null."""
    return _predicate(input, 0, stream)


def is_valid(Column input, stream=None, mr=None):
    """A BOOL8 column without a mask: True where input is valid."""
    return _predicate(input, 1, stream)


def is_nan(Column input, stream=None, mr=None):
    """A BOOL8 column without a mask: True where a FLOAT32 / FLOAT64 input is NaN (a null row is False)."""
    return _predicate(input, 2, stream)


def is_not_nan(Column input, stream=None, mr=None):
    """A BOOL8 column without a mask: True where a FLOAT32 / FLOAT64 input is not NaN (a null row is True)."""
    return _predicate(input, 3, stream)


# ---------------------------------------------------------------------------------------------------------------------
# replacement (python/pylibcudf/pylibcudf/replace.pyx; cpp/include/cudf/replace.hpp)
# ---------------------------------------------------------------------------------------------------------------------
def replace_nulls(Column source_column, replacement, stream=None, mr=None):
    """Nulls of source_column replaced: by replacement[i] (a Column), by one value (a Scalar; the output has no mask), or by the
    nearest valid value before / after the row (a ReplacePolicy; a leading / trailing null run stays null)."""
    from cudf_b200.pylibcudf.replace import ReplacePolicy
    cdef b2_stream s = _stream(stream)
    cdef b2_column* out = NULL
    cdef b2_status st
    cdef Column rc
    cdef const b2_scalar* sc
    cdef int32_t policy
    if isinstance(replacement, Column):
        rc = replacement
        with nogil:
            st = b2_replace_nulls(&source_column.v, &rc.v, s, &out)
    elif isinstance(replacement, _PlcScalar):
        sc = <const b2_scalar*><uintptr_t>replacement._handle
        with nogil:
            st = b2_replace_nulls_scalar(&source_column.v, sc, s, &out)
    elif isinstance(replacement, ReplacePolicy):
        policy = int(replacement)
        with nogil:
            st = b2_replace_nulls_policy(&source_column.v, policy, s, &out)
    else:
        raise TypeError("replacement must be a Column, Scalar, or replace_policy")
    check(st)
    return Column.from_handle(out)


def find_and_replace_all(Column source_column, Column values_to_replace, Column replacement_values, stream=None, mr=None):
    """Rows equal to values_to_replace[j] take replacement_values[j] (the first j among duplicates; -0.0 == +0.0, NaN matches
    nothing)."""
    cdef b2_stream s = _stream(stream)
    cdef b2_column* out = NULL
    cdef b2_status st
    with nogil:
        st = b2_find_and_replace_all(&source_column.v, &values_to_replace.v, &replacement_values.v, s, &out)
    check(st)
    return Column.from_handle(out)


def clamp(Column source_column, lo, hi, lo_replace=None, hi_replace=None, stream=None, mr=None):
    """x < lo -> lo_replace (default lo), x > hi -> hi_replace (default hi); a null bound is not applied."""
    if (lo_replace is None) != (hi_replace is None):
        raise ValueError("lo_replace and hi_replace must be specified together")
    if lo_replace is None:
        lo_replace, hi_replace = lo, hi
    cdef const b2_scalar* l = <const b2_scalar*><uintptr_t>lo._handle
    cdef const b2_scalar* lr = <const b2_scalar*><uintptr_t>lo_replace._handle
    cdef const b2_scalar* h = <const b2_scalar*><uintptr_t>hi._handle
    cdef const b2_scalar* hr = <const b2_scalar*><uintptr_t>hi_replace._handle
    cdef b2_stream s = _stream(stream)
    cdef b2_column* out = NULL
    cdef b2_status st
    with nogil:
        st = b2_clamp(&source_column.v, l, lr, h, hr, s, &out)
    check(st)
    return Column.from_handle(out)


def normalize_nans_and_zeros(Column source_column, bint inplace=False, stream=None, mr=None):
    """Every NaN as quiet_NaN() and -0.0 as +0.0 (FLOAT32 / FLOAT64). inplace=True rewrites source_column's data and returns
    None."""
    cdef b2_stream s = _stream(stream)
    cdef b2_column* out = NULL
    cdef b2_status st
    with nogil:
        if inplace:
            st = b2_normalize_nans_and_zeros_inplace(&source_column.v, s)
        else:
            st = b2_normalize_nans_and_zeros(&source_column.v, s, &out)
    check(st)
    if not inplace:
        return Column.from_handle(out)


# ---------------------------------------------------------------------------------------------------------------------
# joins (python/pylibcudf/pylibcudf/join.pyx:63-205; cudf::hash_join)
# ---------------------------------------------------------------------------------------------------------------------
ctypedef b2_status (*free_join_fn)(const b2_table_view*, const b2_table_view*, int32_t, b2_stream, b2_column**, b2_column**) noexcept nogil


cdef tuple _free_join(free_join_fn fn, Table left_keys, Table right_keys, object nulls_equal, object stream):
    cdef _TableView lv = _TableView.of(left_keys), rv = _TableView.of(right_keys)
    cdef int32_t ne = int(nulls_equal)
    cdef b2_stream s = _stream(stream)
    cdef b2_column* lo = NULL
    cdef b2_column* ro = NULL
    cdef b2_status st
    with nogil:
        st = fn(&lv.tv, &rv.tv, ne, s, &lo, &ro)
    check(st)
    cdef Column l = Column.from_handle(lo)
    return l, Column.from_handle(ro)


def inner_join(Table left_keys, Table right_keys, nulls_equal, stream=None, mr=None):
    return _free_join(b2_inner_join, left_keys, right_keys, nulls_equal, stream)


def left_join(Table left_keys, Table right_keys, nulls_equal, stream=None, mr=None):
    return _free_join(b2_left_join, left_keys, right_keys, nulls_equal, stream)


def full_join(Table left_keys, Table right_keys, nulls_equal, stream=None, mr=None):
    return _free_join(b2_full_join, left_keys, right_keys, nulls_equal, stream)


ctypedef b2_status (*probe_fn)(const b2_hash_join*, const b2_table_view*, int32_t, size_t, b2_stream, b2_column**, b2_column**) noexcept nogil
ctypedef b2_status (*size_fn)(const b2_hash_join*, const b2_table_view*, b2_stream, size_t*) noexcept nogil


cdef class HashJoin:
    """cudf::hash_join (cpp/include/cudf/join/hash_join.hpp): build once, probe many."""
    cdef b2_hash_join* hj
    cdef object build

    def __cinit__(self):
        self.hj = NULL

    def __init__(self, Table build, compare_nulls=0, has_nulls=None, double load_factor=0.5, stream=None):
        cdef _TableView bv = _TableView.of(build)
        cdef int32_t hn = -1 if has_nulls is None else int(bool(has_nulls))
        cdef int32_t cn = int(compare_nulls)
        cdef b2_stream s = _stream(stream)
        cdef b2_status st
        self.build = build
        with nogil:
            st = b2_hash_join_create(&bv.tv, hn, cn, load_factor, s, &self.hj)
        check(st)

    def __dealloc__(self):
        if self.hj != NULL:
            b2_hash_join_destroy(self.hj)
            self.hj = NULL

    cdef tuple _probe(self, probe_fn fn, Table probe, object output_size, object stream):
        cdef _TableView pv = _TableView.of(probe)
        cdef int32_t has = 0 if output_size is None else 1
        cdef size_t osz = int(output_size or 0)
        cdef b2_stream s = _stream(stream)
        cdef b2_column* lo = NULL
        cdef b2_column* ro = NULL
        cdef b2_status st
        with nogil:
            st = fn(self.hj, &pv.tv, has, osz, s, &lo, &ro)
        check(st)
        cdef Column l = Column.from_handle(lo)
        return l, Column.from_handle(ro)

    cdef size_t _size(self, size_fn fn, Table probe, object stream) except? 0:
        cdef _TableView pv = _TableView.of(probe)
        cdef b2_stream s = _stream(stream)
        cdef size_t out = 0
        cdef b2_status st
        with nogil:
            st = fn(self.hj, &pv.tv, s, &out)
        check(st)
        return out

    def inner_join(self, Table probe, output_size=None, stream=None):
        return self._probe(b2_hash_join_inner_join, probe, output_size, stream)

    def left_join(self, Table probe, output_size=None, stream=None):
        return self._probe(b2_hash_join_left_join, probe, output_size, stream)

    def full_join(self, Table probe, output_size=None, stream=None):
        return self._probe(b2_hash_join_full_join, probe, output_size, stream)

    def inner_join_size(self, Table probe, stream=None):
        return self._size(b2_hash_join_inner_join_size, probe, stream)

    def left_join_size(self, Table probe, stream=None):
        return self._size(b2_hash_join_left_join_size, probe, stream)

    def full_join_size(self, Table probe, stream=None):
        return self._size(b2_hash_join_full_join_size, probe, stream)

    # ---- match context / partitioned probes (hash_join.hpp:254-440); implemented below the class ----
    def inner_join_match_context(self, Table probe, stream=None):
        return hash_join_match_context(self, 0, probe, stream)

    def left_join_match_context(self, Table probe, stream=None):
        return hash_join_match_context(self, 1, probe, stream)

    def full_join_match_context(self, Table probe, stream=None):
        return hash_join_match_context(self, 2, probe, stream)

    def partitioned_inner_join(self, context, stream=None):
        return hash_join_partitioned(self, 0, context, stream)

    def partitioned_left_join(self, context, stream=None):
        return hash_join_partitioned(self, 1, context, stream)

    def partitioned_full_join(self, context, stream=None):
        """Probe side only; finalize_partitioned_full_join appends the unmatched build rows."""
        return hash_join_partitioned(self, 2, context, stream)

    @staticmethod
    def finalize_partitioned_full_join(left_partials, right_partials, left_table_num_rows, right_table_num_rows, stream=None):
        return finalize_partitioned_full_join(left_partials, right_partials, left_table_num_rows, right_table_num_rows, stream)


ctypedef b2_status (*filtered_probe_fn)(const b2_filtered_join*, const b2_table_view*, b2_stream, b2_column**) noexcept nogil


cdef class FilteredJoin:
    """cudf::filtered_join (cpp/include/cudf/join/filtered_join.hpp): the right (filter) table's keys become a distinct set
    once; semi_join / anti_join return the ascending INT32 indices of the left rows with / without an equal right row."""
    cdef b2_filtered_join* fj
    cdef object right

    def __cinit__(self):
        self.fj = NULL

    def __init__(self, Table right, compare_nulls, double load_factor=0.5, stream=None):
        cdef _TableView rv = _TableView.of(right)
        cdef int32_t cn = int(compare_nulls)
        cdef b2_stream s = _stream(stream)
        cdef b2_status st
        self.right = right  # keys wider than 8 bytes are compared against its columns
        with nogil:
            st = b2_filtered_join_create(&rv.tv, cn, load_factor, s, &self.fj)
        check(st)

    def __dealloc__(self):
        if self.fj != NULL:
            b2_filtered_join_destroy(self.fj)
            self.fj = NULL

    cdef Column _probe(self, filtered_probe_fn fn, Table left, object stream):
        cdef _TableView lv = _TableView.of(left)
        cdef b2_stream s = _stream(stream)
        cdef b2_column* out = NULL
        cdef b2_status st
        with nogil:
            st = fn(self.fj, &lv.tv, s, &out)
        check(st)
        return Column.from_handle(out)

    def semi_join(self, Table left, stream=None, mr=None):
        return self._probe(b2_filtered_join_semi_join, left, stream)

    def anti_join(self, Table left, stream=None, mr=None):
        return self._probe(b2_filtered_join_anti_join, left, stream)


def left_semi_join(Table left_keys, Table right_keys, nulls_equal, stream=None, mr=None):
    """join.pyx:207-256: a FilteredJoin of `right_keys` probed once."""
    return FilteredJoin(right_keys, nulls_equal, stream=stream).semi_join(left_keys, stream)


def left_anti_join(Table left_keys, Table right_keys, nulls_equal, stream=None, mr=None):
    """join.pyx:259-306: a FilteredJoin of `right_keys` probed once."""
    return FilteredJoin(right_keys, nulls_equal, stream=stream).anti_join(left_keys, stream)


# ---------------------------------------------------------------------------------------------------------------------
# groupby (python/pylibcudf/pylibcudf/groupby.pyx:36-243)
# ---------------------------------------------------------------------------------------------------------------------
cdef class GroupByRequest:
    cdef public Column _values
    cdef public list _aggregations

    def __init__(self, Column values, aggregations):
        self._values = values
        self._aggregations = list(aggregations)


ctypedef b2_status (*groupby_fn)(b2_groupby*, const b2_agg_request*, int32_t, b2_stream, b2_table**, b2_table**) noexcept nogil


cdef class GroupBy:
    cdef b2_groupby* gb
    cdef object keys        # keeps the key buffers alive (groupby.pyx:136-138)
    cdef _TableView kv

    def __cinit__(self):
        self.gb = NULL

    def __init__(self, Table keys, null_handling=NullPolicy.EXCLUDE, keys_are_sorted=Sorted.NO, column_order=None, null_precedence=None):
        self.keys = keys
        self.kv = _TableView.of(keys)
        cdef _Flags o = _Flags.of(column_order), p = _Flags.of(null_precedence)
        cdef int32_t nh = int(null_handling), ks = int(keys_are_sorted)
        cdef b2_status st
        with nogil:
            st = b2_groupby_create(&self.kv.tv, nh, ks, o.p, o.n, p.p, p.n, &self.gb)
        check(st)

    def __dealloc__(self):
        if self.gb != NULL:
            b2_groupby_destroy(self.gb)
            self.gb = NULL

    cdef tuple _run(self, groupby_fn fn, list requests, object stream):
        cdef Py_ssize_t n = len(requests), i, j, m, total = 0
        cdef GroupByRequest r
        for r in requests:
            total += len(r._aggregations)
        cdef b2_agg_request* arr = <b2_agg_request*>calloc(n if n > 0 else 1, sizeof(b2_agg_request))
        cdef int32_t* kinds = <int32_t*>calloc(total if total > 0 else 1, sizeof(int32_t))
        cdef b2_stream s = _stream(stream)
        cdef b2_table* ko = NULL
        cdef b2_table* ro = NULL
        cdef b2_status st
        cdef Py_ssize_t k = 0
        if arr == NULL or kinds == NULL:
            free(arr)
            free(kinds)
            raise MemoryError()
        try:
            for i in range(n):
                r = <GroupByRequest>requests[i]
                m = len(r._aggregations)
                arr[i].values = r._values.v
                arr[i].kinds = kinds + k
                arr[i].num_kinds = <int32_t>m
                for j in range(m):
                    kinds[k + j] = <int32_t>r._aggregations[j].abi_kind()
                k += m
            with nogil:
                st = fn(self.gb, arr, <int32_t>n, s, &ko, &ro)
            check(st)
        finally:
            free(arr)
            free(kinds)
        cdef Table keys = Table.from_handle(ko)
        cdef list flat = Table.from_handle(ro).cols
        cdef list results = []
        k = 0
        for r in requests:
            m = len(r._aggregations)
            results.append(Table(flat[k: k + m]))
            k += m
        return keys, results

    def aggregate(self, requests, stream=None, mr=None):
        """-> (Table group_keys, [Table results per request])  (groupby.pyx:165-201)"""
        return self._run(b2_groupby_aggregate, list(requests), stream)

    def scan(self, requests, stream=None, mr=None):
        return self._run(b2_groupby_scan, list(requests), stream)


# ---------------------------------------------------------------------------------------------------------------------
# reduce / scan / segmented_reduce (python/pylibcudf/pylibcudf/reduce.pyx:48-157)
# ---------------------------------------------------------------------------------------------------------------------
def reduce(Column col, agg, data_type, init=None, stream=None, mr=None):
    """-> Scalar (the ctypes twin's class over the returned b2_scalar handle)."""
    cdef int32_t kind = int(agg.kind()), tid = int(data_type.id())
    cdef const b2_scalar* ini = <const b2_scalar*><uintptr_t>(init._handle if init is not None else 0)
    cdef b2_stream s = _stream(stream)
    cdef b2_scalar* out = NULL
    cdef b2_status st
    with nogil:
        st = b2_reduce(&col.v, kind, tid, ini, s, &out)
    check(st)
    return _PlcScalar(<uintptr_t>out)


def scan(Column col, agg, inclusive, null_handling=NullPolicy.EXCLUDE, stream=None, mr=None):
    cdef int32_t kind = int(agg.kind()), inc = int(inclusive), nh = int(null_handling)
    cdef b2_stream s = _stream(stream)
    cdef b2_column* out = NULL
    cdef b2_status st
    with nogil:
        st = b2_scan(&col.v, kind, inc, nh, s, &out)
    check(st)
    return Column.from_handle(out)


def segmented_reduce(Column segmented_values, Column offsets, agg, data_type, null_handling=NullPolicy.EXCLUDE, init=None, stream=None,
                     mr=None):
    """cudf::segmented_reduce (cpp/include/cudf/reduction.hpp); `offsets` is an INT32 device column."""
    cdef int32_t kind = int(agg.kind()), tid = int(data_type.id()), nh = int(null_handling)
    cdef const int32_t* optr = <const int32_t*>offsets.v.data
    if optr != NULL:
        optr += offsets.v.offset
    cdef int32_t nof = offsets.v.size
    cdef const b2_scalar* ini = <const b2_scalar*><uintptr_t>(init._handle if init is not None else 0)
    cdef b2_stream s = _stream(stream)
    cdef b2_column* out = NULL
    cdef b2_status st
    with nogil:
        st = b2_segmented_reduce(&segmented_values.v, optr, nof, kind, tid, nh, ini, s, &out)
    check(st)
    return Column.from_handle(out)


# ---------------------------------------------------------------------------------------------------------------------
# sorting: segmented sort / top-k / rank (python/pylibcudf/pylibcudf/sorting.pyx; cpp/include/cudf/sorting.hpp:165-416)
# ---------------------------------------------------------------------------------------------------------------------
cdef Column _segmented_sorted_order(Table keys, Column segment_offsets, object column_order, object null_precedence, int stable, object stream):
    cdef _TableView kv = _TableView.of(keys)
    cdef _Flags o = _Flags.of(column_order), p = _Flags.of(null_precedence)
    cdef b2_stream s = _stream(stream)
    cdef b2_column* out = NULL
    cdef b2_status st
    with nogil:
        st = b2_segmented_sorted_order(&kv.tv, &segment_offsets.v, o.p, o.n, p.p, p.n, stable, s, &out)
    check(st)
    return Column.from_handle(out)


cdef Table _segmented_sort_by_key(Table values, Table keys, Column segment_offsets, object column_order, object null_precedence, int stable,
                                  object stream):
    cdef _TableView vv = _TableView.of(values), kv = _TableView.of(keys)
    cdef _Flags o = _Flags.of(column_order), p = _Flags.of(null_precedence)
    cdef b2_stream s = _stream(stream)
    cdef b2_table* out = NULL
    cdef b2_status st
    with nogil:
        st = b2_segmented_sort_by_key(&vv.tv, &kv.tv, &segment_offsets.v, o.p, o.n, p.p, p.n, stable, s, &out)
    check(st)
    return Table.from_handle(out)


def segmented_sorted_order(Table keys, Column segment_offsets, column_order, null_precedence, stream=None, mr=None):
    return _segmented_sorted_order(keys, segment_offsets, column_order, null_precedence, 0, stream)


def stable_segmented_sorted_order(Table keys, Column segment_offsets, column_order, null_precedence, stream=None, mr=None):
    return _segmented_sorted_order(keys, segment_offsets, column_order, null_precedence, 1, stream)


def segmented_sort_by_key(Table values, Table keys, Column segment_offsets, column_order, null_precedence, stream=None, mr=None):
    return _segmented_sort_by_key(values, keys, segment_offsets, column_order, null_precedence, 0, stream)


def stable_segmented_sort_by_key(Table values, Table keys, Column segment_offsets, column_order, null_precedence, stream=None, mr=None):
    return _segmented_sort_by_key(values, keys, segment_offsets, column_order, null_precedence, 1, stream)


ctypedef b2_status (*topk_fn)(const b2_column_view*, int32_t, int32_t, b2_stream, b2_column**) noexcept nogil


cdef Column _top_k(topk_fn fn, Column col, int32_t k, int32_t sort_order, object stream):
    cdef b2_stream s = _stream(stream)
    cdef b2_column* out = NULL
    cdef b2_status st
    with nogil:
        st = fn(&col.v, k, sort_order, s, &out)
    check(st)
    return Column.from_handle(out)


def top_k(Column col, int k, sort_order=1, stream=None, mr=None):
    """cudf::top_k (sorting.hpp:370-391); sort_order defaults to DESCENDING (high to low)."""
    return _top_k(b2_top_k, col, k, int(sort_order), stream)


def top_k_order(Column col, int k, sort_order=1, stream=None, mr=None):
    return _top_k(b2_top_k_order, col, k, int(sort_order), stream)


def rank(Column input_view, method, column_order, null_handling, null_precedence, percentage, stream=None, mr=None):
    """cudf::rank (sorting.hpp:165-230); method: RankMethod (0 FIRST, 1 AVERAGE, 2 MIN, 3 MAX, 4 DENSE)."""
    cdef int32_t m = int(method), co = int(column_order), nh = int(null_handling), npr = int(null_precedence), pct = 1 if percentage else 0
    cdef b2_stream s = _stream(stream)
    cdef b2_column* out = NULL
    cdef b2_status st
    with nogil:
        st = b2_rank(&input_view.v, m, co, nh, npr, pct, s, &out)
    check(st)
    return Column.from_handle(out)


# ---------------------------------------------------------------------------------------------------------------------
# hash_join match contexts / partitioned probes (cpp/include/cudf/join/hash_join.hpp:254-440, join.hpp:81-125)
# ---------------------------------------------------------------------------------------------------------------------
cdef class JoinMatchContext:
    """cudf::join_match_context: the left table and its per-row match counts (INT32 column)."""
    cdef public Table _left_table
    cdef public Column _match_counts
    cdef public int _kind

    def __init__(self, Table left_table, Column match_counts, int kind=0):
        self._left_table = left_table
        self._match_counts = match_counts
        self._kind = kind


cdef class JoinPartitionContext:
    """cudf::join_partition_context (join.hpp:120-125)."""
    cdef public JoinMatchContext left_table_context
    cdef public int left_start_idx
    cdef public int left_end_idx

    def __init__(self, JoinMatchContext left_table_context, int left_start_idx, int left_end_idx):
        self.left_table_context = left_table_context
        self.left_start_idx = left_start_idx
        self.left_end_idx = left_end_idx


def hash_join_match_context(HashJoin hj, int kind, Table probe, stream=None):
    cdef _TableView pv = _TableView.of(probe)
    cdef b2_stream s = _stream(stream)
    cdef b2_column* out = NULL
    cdef b2_status st
    with nogil:
        st = b2_hash_join_match_counts(hj.hj, &pv.tv, kind, s, &out)
    check(st)
    return JoinMatchContext(probe, Column.from_handle(out), kind)


def hash_join_partitioned(HashJoin hj, int kind, JoinPartitionContext context, stream=None):
    cdef JoinMatchContext ctx = context.left_table_context
    if ctx is None or ctx._match_counts is None:
        raise ValueError("join_partition_context without a match context")
    cdef _TableView pv = _TableView.of(ctx._left_table)
    cdef Column counts = ctx._match_counts
    cdef int32_t a = context.left_start_idx, b = context.left_end_idx
    cdef b2_stream s = _stream(stream)
    cdef b2_column* lo = NULL
    cdef b2_column* ro = NULL
    cdef b2_status st
    with nogil:
        st = b2_hash_join_partitioned_join(hj.hj, &pv.tv, &counts.v, a, b, kind, s, &lo, &ro)
    check(st)
    cdef Column l = Column.from_handle(lo)
    return l, Column.from_handle(ro)


def finalize_partitioned_full_join(left_partials, right_partials, int left_table_num_rows, int right_table_num_rows, stream=None):
    cdef list lp = list(left_partials), rp = list(right_partials)
    cdef Py_ssize_t n = len(lp), i
    if len(rp) != n:
        raise ValueError("left and right partials differ in number")
    cdef b2_column_view* lv = <b2_column_view*>calloc(n if n > 0 else 1, sizeof(b2_column_view))
    cdef b2_column_view* rv = <b2_column_view*>calloc(n if n > 0 else 1, sizeof(b2_column_view))
    cdef b2_stream s = _stream(stream)
    cdef b2_column* lo = NULL
    cdef b2_column* ro = NULL
    cdef b2_status st
    if lv == NULL or rv == NULL:
        free(lv)
        free(rv)
        raise MemoryError()
    try:
        for i in range(n):
            lv[i] = (<Column?>lp[i]).v
            rv[i] = (<Column?>rp[i]).v
        with nogil:
            st = b2_hash_join_finalize_full_join(lv, rv, <int32_t>n, left_table_num_rows, right_table_num_rows, s, &lo, &ro)
        check(st)
    finally:
        free(lv)
        free(rv)
    cdef Column l = Column.from_handle(lo)
    return l, Column.from_handle(ro)


# ---------------------------------------------------------------------------------------------------------------------
# partitioning (python/pylibcudf/pylibcudf/partitioning.pyx; cpp/include/cudf/partitioning.hpp:58-175)
# ---------------------------------------------------------------------------------------------------------------------
def hash_partition(Table input, keys, int num_partitions, hash_function=1, seed=0, stream=None, mr=None):  # noqa: A002
    """cudf::hash_partition: `keys` is a Table of key columns or a list of column indices of `input`; libcudf's row hash
    (MurmurHash3_x86_32 per column, hash_combine), partition = hash % num_partitions. -> (table, num_partitions + 1 offsets)."""
    cdef Table ktab
    if isinstance(keys, Table):
        ktab = keys
    else:
        cols = input.cols
        for i in keys:
            if not 0 <= int(i) < len(cols):
                raise IndexError("columns_to_hash: invalid column index")  # std::out_of_range
        ktab = Table([cols[int(i)] for i in keys])
    if ktab.num_columns() and ktab.num_rows() != input.num_rows():
        raise ValueError("Input table and key table must have same number of rows, or key table should have no columns.")
    cdef _TableView tv = _TableView.of(input), kv = _TableView.of(ktab)
    cdef Py_ssize_t noff = (num_partitions if num_partitions > 0 else 0) + 1
    cdef int32_t* offs = <int32_t*>calloc(noff, sizeof(int32_t))
    cdef int32_t hf = int(hash_function)
    cdef uint32_t sd = int(seed) & 0xFFFFFFFF
    cdef b2_stream s = _stream(stream)
    cdef b2_table* out = NULL
    cdef b2_status st
    if offs == NULL:
        raise MemoryError()
    try:
        with nogil:
            st = b2_hash_partition(&tv.tv, &kv.tv, num_partitions, hf, sd, s, &out, offs)
        check(st)
        res = [offs[j] for j in range(noff)]
    finally:
        free(offs)
    return Table.from_handle(out), res


def partition(Table t, Column partition_map, int num_partitions, stream=None, mr=None):
    """cudf::partition (partitioning.hpp:58-101): rows go to the partition their map entry names (stable).
    -> (partitioned table, num_partitions + 1 offsets)."""
    if partition_map.v.null_count > 0:
        raise RuntimeError("Unexpected null values in partition_map.")  # cudf::logic_error
    if num_partitions < 0:
        raise ValueError("num_partitions must not be negative")
    if partition_map.v.size != (t.num_rows() if t.num_columns() else 0):
        raise RuntimeError("Size mismatch between table and partition map.")
    cdef _TableView tv = _TableView.of(t)
    cdef Py_ssize_t noff = num_partitions + 1
    cdef int32_t* offs = <int32_t*>calloc(noff, sizeof(int32_t))
    cdef b2_stream s = _stream(stream)
    cdef b2_table* out = NULL
    cdef b2_status st
    if offs == NULL:
        raise MemoryError()
    try:
        with nogil:
            st = b2_partition_by_map(&tv.tv, &partition_map.v, num_partitions, s, &out, offs)
        check(st)
        res = [offs[j] for j in range(noff)]
    finally:
        free(offs)
    return Table.from_handle(out), res


# ---------------------------------------------------------------------------------------------------------------------
# null masks (python/pylibcudf/pylibcudf/null_mask.pyx; cpp/include/cudf/null_mask.hpp)
# ---------------------------------------------------------------------------------------------------------------------
def _device_buffer(uintptr_t handle):
    from cudf_b200.pylibcudf.null_mask import DeviceBuffer  # owning rmm::device_buffer stand-in of the ctypes twin

    return DeviceBuffer(handle)


def bitmask_allocation_size_bytes(int number_of_bits):
    return int(b2_bitmask_allocation_size_bytes(number_of_bits))


def create_null_mask(int size, state=0, stream=None, mr=None):
    cdef int32_t stt = int(state)
    cdef b2_stream s = _stream(stream)
    cdef b2_buffer* out = NULL
    cdef b2_status st
    with nogil:
        st = b2_create_null_mask(size, stt, s, &out)
    check(st)
    return _device_buffer(<uintptr_t>out)


def copy_bitmask(Column col, stream=None, mr=None):
    cdef b2_stream s = _stream(stream)
    cdef b2_buffer* out = NULL
    cdef b2_status st
    with nogil:
        st = b2_copy_bitmask(col.v.null_mask, col.v.offset, col.v.offset + col.v.size, s, &out)
    check(st)
    return _device_buffer(<uintptr_t>out)


def bitmask_and(columns, stream=None, mr=None):
    cdef Table tbl = columns if isinstance(columns, Table) else Table(columns)
    cdef _TableView tv = _TableView.of(tbl)
    cdef b2_stream s = _stream(stream)
    cdef b2_buffer* out = NULL
    cdef int32_t nc = 0
    cdef b2_status st
    with nogil:
        st = b2_bitmask_and(&tv.tv, s, &out, &nc)
    check(st)
    return _device_buffer(<uintptr_t>out), nc


def null_count(uintptr_t bitmask_ptr, int start, int stop, stream=None):
    cdef b2_stream s = _stream(stream)
    cdef int32_t out = 0
    check(b2_null_count(<const uint32_t*>bitmask_ptr, start, stop, s, &out))
    return out


def count_set_bits(uintptr_t bitmask_ptr, int start, int stop, stream=None):
    cdef b2_stream s = _stream(stream)
    cdef int32_t out = 0
    check(b2_count_set_bits(<const uint32_t*>bitmask_ptr, start, stop, s, &out))
    return out


def set_null_mask(uintptr_t bitmask_ptr, int begin_bit, int end_bit, valid, stream=None):
    cdef b2_stream s = _stream(stream)
    check(b2_set_null_mask(<uint32_t*>bitmask_ptr, begin_bit, end_bit, 1 if valid else 0, s))


# ---------------------------------------------------------------------------------------------------------------------
# contiguous_split: pack / unpack in libcudf's wire format (python/pylibcudf/pylibcudf/contiguous_split.pyx;
# cpp/include/cudf/contiguous_split.hpp:233-317). PackedColumns is the ctypes twin's class.
# ---------------------------------------------------------------------------------------------------------------------
def packed_size(Table input, stream=None):  # noqa: A002
    cdef _TableView tv = _TableView.of(input)
    cdef size_t out = 0
    check(b2_packed_size(&tv.tv, &out))
    return out


def pack(Table input, stream=None, mr=None):  # noqa: A002
    from cudf_b200.pylibcudf.contiguous_split import PackedColumns, _Buffer

    cdef _TableView tv = _TableView.of(input)
    cdef size_t cap = 16 + 40 * len(input.cols), mdsz = 0
    cdef uint8_t* md = <uint8_t*>calloc(cap, 1)
    cdef b2_stream s = _stream(stream)
    cdef b2_buffer* buf = NULL
    cdef b2_status st
    if md == NULL:
        raise MemoryError()
    try:
        with nogil:
            st = b2_pack(&tv.tv, s, md, cap, &mdsz, &buf)
        check(st)
        meta = bytes(md[:mdsz])
    finally:
        free(md)
    owner = _Buffer(<uintptr_t>buf)
    return PackedColumns(meta, <uintptr_t>b2_buffer_data(buf), b2_buffer_size(buf), owner)


def pack_metadata(Table table, uintptr_t contiguous_buffer_ptr, size_t buffer_size):
    cdef _TableView tv = _TableView.of(table)
    cdef size_t cap = 16 + 40 * len(table.cols), mdsz = 0
    cdef uint8_t* md = <uint8_t*>calloc(cap, 1)
    if md == NULL:
        raise MemoryError()
    try:
        check(b2_pack_metadata(&tv.tv, <const uint8_t*>contiguous_buffer_ptr, buffer_size, md, cap, &mdsz))
        return bytes(md[:mdsz])
    finally:
        free(md)


def unpack_from_memoryviews(metadata, uintptr_t gpu_data_ptr, owner=None):
    """cudf::unpack(metadata, gpu_data): the columns of the result point into gpu_data (kept alive through `owner`)."""
    cdef bytes md = bytes(metadata)
    cdef Py_ssize_t n = len(md)
    cdef int32_t ncap = <int32_t>(max(0, (n - 16) // 40) + 1)
    cdef b2_column_view* views = <b2_column_view*>calloc(ncap, sizeof(b2_column_view))
    cdef int32_t ncols = 0, nrows = 0, i
    cdef const uint8_t* mp = <const uint8_t*>md
    cdef list cols = []
    if views == NULL:
        raise MemoryError()
    try:
        check(b2_unpack(mp, <size_t>n, <const void*>gpu_data_ptr, views, ncap, &ncols, &nrows))
        for i in range(ncols):
            cols.append(Column.from_pointers(DataType(TypeId(views[i].type_id)), views[i].size, <uintptr_t>views[i].data,
                                             <uintptr_t>views[i].null_mask, views[i].null_count, 0, [owner]))
    finally:
        free(views)
    return Table(cols)


def unpack(input):  # noqa: A002
    return unpack_from_memoryviews(input.metadata, input.gpu_data_ptr, input)
