"""cudf stream compaction semantics (cpp/src/stream_compaction/{apply_boolean_mask,drop_nulls,drop_nans,unique,distinct}.cu).

Columns are (values, valid | None) pairs. Key rows compare with the normalisation the sort and groupby oracles use:
-0 == +0, every NaN equals every NaN (unless nans_equal is UNEQUAL), null == null (unless nulls_equal is UNEQUAL).
keep: 0 ANY, 1 FIRST, 2 LAST, 3 NONE."""
from __future__ import annotations

import numpy as np

KEEP_ANY, KEEP_FIRST, KEEP_LAST, KEEP_NONE = 0, 1, 2, 3


def _valid(col):
    v, m = col
    return np.ones(len(v), bool) if m is None else np.asarray(m, bool)


def gather(cols, idx):
    idx = np.asarray(idx, dtype=np.int64)
    return [(np.asarray(v)[idx], None if m is None else np.asarray(m, bool)[idx]) for v, m in cols]


def _rows(cols, mask):
    return gather(cols, np.flatnonzero(mask))


def apply_boolean_mask(cols, mask, deletion=False):
    mv, mm = mask
    if len(mv) == 0 or (cols and len(cols[0][0]) == 0):
        return gather(cols, [])
    keep = _valid(mask) & ((np.asarray(mv) != 0) != deletion)
    return _rows(cols, keep)


def drop_nulls(cols, keys, keep_threshold=None):
    thr = len(keys) if keep_threshold is None else keep_threshold
    # no keys, no rows or no nulls in the keys: a copy, whatever the threshold (drop_nulls.cu:57-60)
    if not keys or len(cols[0][0]) == 0 or all(_valid(cols[k]).all() for k in keys):
        return gather(cols, np.arange(len(cols[0][0]) if cols else 0))
    cnt = sum(_valid(cols[k]).astype(np.int64) for k in keys)
    return _rows(cols, cnt >= thr)


def drop_nans(cols, keys, keep_threshold=None):
    thr = len(keys) if keep_threshold is None else keep_threshold
    if not keys or len(cols[0][0]) == 0:
        return gather(cols, np.arange(len(cols[0][0]) if cols else 0))
    for k in keys:
        if np.asarray(cols[k][0]).dtype.kind != "f":
            raise RuntimeError("Key column is not of type floating-point")
    cnt = sum((~_valid(cols[k]) | ~np.isnan(cols[k][0])).astype(np.int64) for k in keys)
    return _rows(cols, cnt >= thr)


def _row_keys(keycols, nulls_equal=0, nans_equal=0):
    """One hashable token per row; rows that equal no other row get a unique token."""
    n = len(keycols[0][0])
    parts = []
    lonely = np.zeros(n, bool)
    for v, m in keycols:
        v = np.asarray(v)
        valid = np.ones(n, bool) if m is None else np.asarray(m, bool)
        if v.dtype.kind == "f":
            nan = np.isnan(v)
            vals = np.where(v == 0, 0.0, v).astype(np.float64)
            toks = [("nan",) if nn else float(x) for x, nn in zip(vals.tolist(), nan.tolist())]
            if nans_equal:
                lonely |= nan & valid
        else:
            toks = v.tolist()
        toks = [t if ok else ("null",) for t, ok in zip(toks, valid.tolist())]
        if nulls_equal:
            lonely |= ~valid
        parts.append(toks)
    rows = list(zip(*parts))
    return [("lonely", i) if lonely[i] else rows[i] for i in range(n)]


def unique_indices(keycols, keep, nulls_equal=0):
    keep = KEEP_FIRST if keep == KEEP_ANY else keep
    n = len(keycols[0][0])
    rk = _row_keys(keycols, nulls_equal, 0)
    out = []
    for i in range(n):
        dup_prev = i > 0 and rk[i] == rk[i - 1]
        dup_next = i + 1 < n and rk[i] == rk[i + 1]
        if keep == KEEP_FIRST and dup_prev or keep == KEEP_LAST and dup_next or keep == KEEP_NONE and (dup_prev or dup_next):
            continue
        out.append(i)
    return np.asarray(out, dtype=np.int32)


def unique(cols, keys, keep, nulls_equal=0):
    if not cols or len(cols[0][0]) == 0 or not keys:
        return gather(cols, [])
    return gather(cols, unique_indices([cols[k] for k in keys], keep, nulls_equal))


def distinct_indices(keycols, keep, nulls_equal=0, nans_equal=0):
    """Ascending indices of the kept rows. ANY keeps the first row of each set (one valid choice of the reference's any)."""
    if not keycols or len(keycols[0][0]) == 0:
        return np.zeros(0, np.int32)
    rk = _row_keys(keycols, nulls_equal, nans_equal)
    first, last, count = {}, {}, {}
    for i, k in enumerate(rk):
        first.setdefault(k, i)
        last[k] = i
        count[k] = count.get(k, 0) + 1
    if keep in (KEEP_ANY, KEEP_FIRST):
        idx = list(first.values())
    elif keep == KEEP_LAST:
        idx = list(last.values())
    else:
        idx = [first[k] for k, c in count.items() if c == 1]
    return np.sort(np.asarray(idx, dtype=np.int32))


def stable_distinct(cols, keys, keep, nulls_equal=0, nans_equal=0):
    if not cols or len(cols[0][0]) == 0 or not keys:
        return gather(cols, [])
    return gather(cols, distinct_indices([cols[k] for k in keys], keep, nulls_equal, nans_equal))
