"""Left semi / anti join semantics (cpp/src/join/filtered_join/filtered_join.cu:124-186 of the reference) restated on the
hash join oracle's row ids (oracle/join.py `_row_ids`): a left row is in the semi result when its id is >= 0 and occurs among
the right ids, in the anti result otherwise. Results are INT32 and ascending."""
from __future__ import annotations

import numpy as np

from oracle.join import EQUAL, UNEQUAL, _row_ids  # noqa: F401  (EQUAL / UNEQUAL re-exported for the tests)


def _rows(cols) -> int:
    return len(cols[0][0]) if cols else 0


def _check_shape(left_cols, right_cols):
    """check_shape_compatibility: a column count or type mismatch is std::invalid_argument."""
    if len(left_cols) != len(right_cols):
        raise ValueError("Mismatch in number of columns to be joined on")
    for (lv, _), (rv, _) in zip(left_cols, right_cols):
        if np.asarray(lv).dtype != np.asarray(rv).dtype:
            raise ValueError("Mismatch in joining column data types")


def contains(left_cols, right_cols, nulls_equal=EQUAL) -> np.ndarray:
    """Per left row: does some right row equal it (both sides non-empty)."""
    _check_shape(left_cols, right_cols)
    if len(left_cols) == 1 and left_cols[0][1] is None and right_cols[0][1] is None and np.asarray(left_cols[0][0]).dtype.kind in "iu":
        return np.isin(left_cols[0][0], right_cols[0][0])  # one integer key without nulls: value membership
    lid, rid = _row_ids(left_cols, right_cols, nulls_equal)
    return (lid >= 0) & np.isin(lid, rid[rid >= 0])


def left_semi_join(left_cols, right_cols, nulls_equal=EQUAL) -> np.ndarray:
    if _rows(left_cols) == 0 or _rows(right_cols) == 0:
        return np.empty(0, np.int32)
    return np.nonzero(contains(left_cols, right_cols, nulls_equal))[0].astype(np.int32)


def left_anti_join(left_cols, right_cols, nulls_equal=EQUAL) -> np.ndarray:
    n = _rows(left_cols)
    if n == 0:
        return np.empty(0, np.int32)
    if _rows(right_cols) == 0:
        return np.arange(n, dtype=np.int32)
    return np.nonzero(~contains(left_cols, right_cols, nulls_equal))[0].astype(np.int32)
