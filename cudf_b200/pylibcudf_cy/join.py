"""pylibcudf.join (python/pylibcudf/pylibcudf/join.pyx:63-306) + cudf::hash_join with its match contexts and cudf::filtered_join:
compiled in _core.pyx."""
from ._core import (FilteredJoin, HashJoin, JoinMatchContext, JoinPartitionContext, full_join, inner_join, left_anti_join, left_join,
                    left_semi_join)

__all__ = ["inner_join", "left_join", "full_join", "left_semi_join", "left_anti_join", "HashJoin", "FilteredJoin", "JoinMatchContext",
           "JoinPartitionContext"]
