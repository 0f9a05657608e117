"""pylibcudf.replace (python/pylibcudf/pylibcudf/replace.pyx; cpp/include/cudf/replace.hpp): compiled in _core.pyx."""
from ..pylibcudf.replace import ReplacePolicy
from ._core import clamp, find_and_replace_all, normalize_nans_and_zeros, replace_nulls

__all__ = ["ReplacePolicy", "clamp", "find_and_replace_all", "normalize_nans_and_zeros", "replace_nulls"]
