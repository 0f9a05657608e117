"""pylibcudf.binaryop (python/pylibcudf/pylibcudf/binaryop.pyx; cpp/include/cudf/binaryop.hpp): compiled in _core.pyx."""
from ..pylibcudf.binaryop import BinaryOperator
from ._core import binary_operation, is_supported_operation

__all__ = ["binary_operation", "is_supported_operation", "BinaryOperator"]
