"""Known answers for the left semi / anti join, transcribed from the reference tree:
cpp/tests/join/semi_anti_join_tests.cpp (file:line in "src") and the examples of cpp/include/cudf/join/filtered_join.hpp.

Each case: "left" / "right" = list of (values with None for null, dtype) columns (an empty list is a table with no columns),
"nulls_equal" (0 EQUAL, 1 UNEQUAL), the expected ascending left indices "semi" and "anti", and "derived": the results the
reference does not state (the anti side of a semi-only test, the UNEQUAL variants), which follow from the semantics."""

CASES = [
    # TestSimple: semi rows {0, 1} (:131); the anti side is derived
    {"src": "semi_anti_join_tests.cpp:117-134", "left": [([0, 1, 2], "int32")], "right": [([0, 1, 3], "int32")],
     "nulls_equal": 0, "semi": [0, 1], "anti": [2], "derived": ["anti"]},
    # PrefilterNullableColumnsNullsEqual, integer inputs: left {1, N, 3, 4, N}, right {N, 3, 5, 6}; under EQUAL the left nulls
    # match the right null
    {"src": "semi_anti_join_tests.cpp:456-487", "left": [([1, None, 3, 4, None], "int32")],
     "right": [([None, 3, 5, 6], "int32")], "nulls_equal": 0, "semi": [1, 2, 4], "anti": [0, 3], "derived": []},
    {"src": "semi_anti_join_tests.cpp:456-487 (UNEQUAL)", "left": [([1, None, 3, 4, None], "int32")],
     "right": [([None, 3, 5, 6], "int32")], "nulls_equal": 1, "semi": [2], "anti": [0, 1, 3, 4], "derived": ["semi", "anti"]},
    # MarkJoinPrefilterLoadFactorOverload's inputs: semi values {1, 1, 3} (:509) are left rows 1, 2, 4
    {"src": "semi_anti_join_tests.cpp:489-518", "left": [([0, 1, 1, 2, 3, 5], "int32")], "right": [([1, 3, 3, 4], "int32")],
     "nulls_equal": 0, "semi": [1, 2, 4], "anti": [0, 3, 5], "derived": ["anti"]},
    # AntiJoinEmptyTables / SemiJoinEmptyTables (cudf::table{} has no columns and no rows)
    {"src": "semi_anti_join_tests.cpp:365-372,398-405 (both empty)", "left": [], "right": [], "nulls_equal": 0,
     "semi": [], "anti": [], "derived": []},
    {"src": "semi_anti_join_tests.cpp:373-380,406-413 (empty right)", "left": [([0, 1, 2], "int32")], "right": [],
     "nulls_equal": 0, "semi": [], "anti": [0, 1, 2], "derived": []},
    {"src": "semi_anti_join_tests.cpp:381-388,414-421 (empty left)", "left": [], "right": [([0, 1, 2], "int32")],
     "nulls_equal": 0, "semi": [], "anti": [], "derived": []},
    # filtered_join.hpp doc examples: right (filter) {1, 2, 3}, left {0, 1, 2}
    {"src": "filtered_join.hpp:107-111", "left": [([0, 1, 2], "int32")], "right": [([1, 2, 3], "int32")], "nulls_equal": 0,
     "semi": [1, 2], "anti": [0], "derived": ["anti"]},
    {"src": "filtered_join.hpp:132-136", "left": [([0, 1, 2], "int32")], "right": [([1, 2, 3], "int32")], "nulls_equal": 0,
     "semi": [1, 2], "anti": [0], "derived": ["semi"]},
]

# InvalidLoadFactor (semi_anti_join_tests.cpp:520-532): filtered_join(table {0, 1, 2}, EQUAL, lf) throws std::invalid_argument
INVALID_LOAD_FACTORS = {"src": "semi_anti_join_tests.cpp:520-532", "right": [([0, 1, 2], "int32")], "load_factors": [-0.1, 0.0, 1.1]}
