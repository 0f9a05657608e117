"""pylibcudf.unary (python/pylibcudf/pylibcudf/unary.pyx; cpp/include/cudf/unary.hpp): compiled in _core.pyx."""
from ..pylibcudf.unary import UnaryOperator
from ._core import bit_cast, cast, is_nan, is_not_nan, is_null, is_supported_cast, is_valid, unary_operation

__all__ = ["UnaryOperator", "unary_operation", "is_null", "is_valid", "cast", "is_supported_cast", "bit_cast", "is_nan", "is_not_nan"]
