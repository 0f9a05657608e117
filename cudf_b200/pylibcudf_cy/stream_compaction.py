"""pylibcudf.stream_compaction (python/pylibcudf/pylibcudf/stream_compaction.pyx; cpp/include/cudf/stream_compaction.hpp): compiled in
_core.pyx."""
from ..pylibcudf.stream_compaction import DuplicateKeepOption
from ._core import (apply_boolean_mask, apply_deletion_mask, distinct, distinct_indices, drop_nans, drop_nulls, stable_distinct,
                    unique)

__all__ = ["apply_boolean_mask", "apply_deletion_mask", "distinct", "distinct_indices", "drop_nans", "drop_nulls", "stable_distinct",
           "unique", "DuplicateKeepOption"]
