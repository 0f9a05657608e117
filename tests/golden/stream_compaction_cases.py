"""Fixed-width known-answer cases of cpp/tests/stream_compaction/*_tests.cpp (reference tree), transcribed with their
file:line. A value of None is a null. Columns are (values, dtype); `expected` is the table the reference test compares
against (values under nulls are not compared). The reference sorts a `distinct` result before comparing it, so `distinct`
cases are compared after a canonical row sort; every other operation is compared in order. keep: 0 ANY, 1 FIRST, 2 LAST,
3 NONE; nulls_equal: 0 EQUAL, 1 UNEQUAL; nans_equal: 0 ALL_EQUAL, 1 UNEQUAL."""
import math

NAN = math.nan
I16, I32, F32, F64, B8 = "int16", "int32", "float32", "float64", "bool"

_MASK_TABLE = [([True, False, None, False, True, None], I16), ([10, 40, None, 5, 2, None], I32),
               ([10.0, 40.0, None, 5.0, 2.0, None], F64)]
_UNIQUE_TABLE = [([5, None, 3, 2, 5, 8, 1], I32), ([20, 20, None, None, 19, 21, 19], I32)]
_NAN_TABLE = [([1.0, 2.0, None, NAN, 5.0, None], F32), ([10, 40, None, 5, 2, None], I32),
              ([NAN, 40.0, None, 5.0, 2.0, None], F64)]

CASES = [
    dict(src="apply_boolean_mask_tests.cpp:36-52", op="apply_boolean_mask", table=_MASK_TABLE,
         mask=([True, False, True, False, True, False], B8),
         expected=[([True, None, True], I16), ([10, None, 2], I32), ([10.0, None, 2.0], F64)]),
    dict(src="apply_boolean_mask_tests.cpp:54-70", op="apply_boolean_mask", table=_MASK_TABLE,
         mask=([None, False, True, False, True, False], B8),
         expected=[([None, True], I16), ([None, 2], I32), ([None, 2.0], F64)]),
    dict(src="drop_nans_tests.cpp:19-42", op="drop_nans", table=_NAN_TABLE, keys=[0, 2], threshold=None,
         expected=[([2.0, None, 5.0, None], F32), ([40, None, 2, None], I32), ([40.0, None, 2.0, None], F64)]),
    dict(src="drop_nans_tests.cpp:60-83", op="drop_nans",
         table=[([1.0, 2.0, None, NAN, 5.0, None], F32), ([10, 40, None, 5, 2, None], I32),
                ([NAN, 40.0, None, NAN, 2.0, None], F64)], keys=[0, 2], threshold=1,
         expected=[([1.0, 2.0, None, 5.0, None], F32), ([10, 40, None, 2, None], I32), ([NAN, 40.0, None, 2.0, None], F64)]),
    dict(src="unique_tests.cpp:137-152", op="unique", table=_UNIQUE_TABLE, keys=[1], keep=1, nulls_equal=0,
         expected=[([5, 3, 5, 8, 1], I32), ([20, None, 19, 21, 19], I32)]),
    dict(src="unique_tests.cpp:154-167", op="unique", table=_UNIQUE_TABLE, keys=[1], keep=1, nulls_equal=1,
         expected=[([5, 3, 2, 5, 8, 1], I32), ([20, None, None, 19, 21, 19], I32)]),
    dict(src="unique_tests.cpp:169-184", op="unique", table=_UNIQUE_TABLE, keys=[1], keep=2, nulls_equal=0,
         expected=[([None, 2, 5, 8, 1], I32), ([20, None, 19, 21, 19], I32)]),
    dict(src="unique_tests.cpp:186-199", op="unique", table=_UNIQUE_TABLE, keys=[1], keep=2, nulls_equal=1,
         expected=[([None, 3, 2, 5, 8, 1], I32), ([20, None, None, 19, 21, 19], I32)]),
    dict(src="unique_tests.cpp:201-216", op="unique", table=_UNIQUE_TABLE, keys=[1], keep=3, nulls_equal=0,
         expected=[([5, 8, 1], I32), ([19, 21, 19], I32)]),
    dict(src="unique_tests.cpp:218-231", op="unique", table=_UNIQUE_TABLE, keys=[1], keep=3, nulls_equal=1,
         expected=[([3, 2, 5, 8, 1], I32), ([None, None, 19, 21, 19], I32)]),
]

_DN_TABLE = [([True, False, None, False, True, None], I16), ([10, 40, None, 5, 2, None], I32), ([10.0, 40.0, None, 5.0, 2.0, None], F64)]
_DN_EXP = [([True, False, False, True], I16), ([10, 40, 5, 2], I32), ([10.0, 40.0, 5.0, 2.0], F64)]
_ALL5 = [([1, 2, 3, 4, 5], I32)]
_DEL_EXP = [([False, False, None], I16), ([40, 5, None], I32), ([40.0, 5.0, None], F64)]
CASES += [
    dict(src="drop_nulls_tests.cpp:21-42", op="drop_nulls", table=_DN_TABLE, keys=[0, 1, 2], threshold=None, expected=_DN_EXP),
    dict(src="drop_nulls_tests.cpp:44-58", op="drop_nulls",
         table=[([True, False, True, False, True, False], I16), ([10, 40, 70, 5, 2, 10], I32), ([10.0, 40.0, 70.0, 5.0, 2.0, 10.0], F64)],
         keys=[0, 1, 2], threshold=None,
         expected=[([True, False, True, False, True, False], I16), ([10, 40, 70, 5, 2, 10], I32), ([10.0, 40.0, 70.0, 5.0, 2.0, 10.0], F64)]),
    dict(src="drop_nulls_tests.cpp:60-81", op="drop_nulls",
         table=[([True, False, None, False, True, None], I16), ([10, 40, None, 5, 2, None], I32), ([10.0, 40.0, None, 5.0, 2.0, 10.0], F64)],
         keys=[0, 1, 2], threshold=None, expected=_DN_EXP),
    dict(src="drop_nulls_tests.cpp:129-150", op="drop_nulls",
         table=[([True, False, None, False, True, None], I16), ([10, 40, None, 5, 2, 10], I32), ([10.0, 40.0, 70.0, 5.0, 2.0, 10.0], F64)],
         keys=[0, 1, 2], threshold=2,
         expected=[([True, False, False, True, None], I16), ([10, 40, 5, 2, 10], I32), ([10.0, 40.0, 5.0, 2.0, 10.0], F64)]),
    dict(src="drop_nulls_tests.cpp:180-189", op="drop_nulls", table=_DN_TABLE, keys=[], threshold=None, expected=_DN_TABLE),
    dict(src="apply_boolean_mask_tests.cpp:372-389", op="apply_deletion_mask", table=_MASK_TABLE,
         mask=([True, False, True, False, True, False], B8), expected=_DEL_EXP),
    dict(src="apply_boolean_mask_tests.cpp:391-408", op="apply_deletion_mask", table=_MASK_TABLE,
         mask=([None, False, True, False, True, False], B8), expected=_DEL_EXP),
    dict(src="apply_boolean_mask_tests.cpp:449-460", op="apply_deletion_mask", table=_ALL5, mask=([True] * 5, B8),
         expected=[([], I32)]),
    dict(src="apply_boolean_mask_tests.cpp:462-473", op="apply_deletion_mask", table=_ALL5, mask=([False] * 5, B8), expected=_ALL5),
    dict(src="apply_boolean_mask_tests.cpp:475-487", op="apply_deletion_mask", table=_ALL5,
         mask=([True, True, True, None, None], B8), expected=[([], I32)]),
]

# distinct_tests.cpp:165-204 (KEEP_ANY; rows with equal keys are equal rows)
_NAN_ANY = [([6, 6, 6, 1, 1, 1, 3, 5, 8, 5], I32), ([6.0, 6, 6, 1, 1, 1, 3, 4, 9, 4], F32),
            ([20, 20, 20, 15, 15, 15, 20, 19, 21, 9], I32), ([19.0, 19, 19, NAN, NAN, NAN, 20, 20, 9, 21], F32)]
CASES += [
    dict(src="distinct_tests.cpp:165-186", op="distinct", table=_NAN_ANY, keys=[2, 3], keep=0, nulls_equal=0, nans_equal=1,
         expected=[([5, 1, 1, 1, 5, 6, 3, 8], I32), ([4.0, 1, 1, 1, 4, 6, 3, 9], F32), ([9, 15, 15, 15, 19, 20, 20, 21], I32),
                   ([21.0, NAN, NAN, NAN, 20, 19, 20, 9], F32)]),
    dict(src="distinct_tests.cpp:188-203", op="distinct", table=_NAN_ANY, keys=[2, 3], keep=0, nulls_equal=0, nans_equal=0,
         expected=[([5, 1, 5, 6, 3, 8], I32), ([4.0, 1, 4, 6, 3, 9], F32), ([9, 15, 19, 20, 20, 21], I32),
                   ([21.0, NAN, 20, 19, 20, 9], F32)]),
]

# distinct_tests.cpp:437-603 and stable_distinct_tests.cpp:404-559 run the same inputs; the stable results are the distinct
# results in input order (column 0 is the row id)
_NULLS_EQ = [([0, 1, 2, 3, 4, 5, 6], I32), ([20, None, None, 19, 21, 19, 22], I32)]
_NULLS_NE = [([0, 1, 2, 3, 4, 5, 6, 7], I32), ([20, None, None, 19, 21, 19, 22, 20], I32)]
_NANS_EQ = [([0, 1, 2, 3, 4, 5, 6], I32), ([20.0, NAN, NAN, 19, 21, 19, 22], F32)]
_NANS_NE = [([0, 1, 2, 3, 4, 5, 6, 7], I32), ([20.0, NAN, NAN, 19, 21, 19, 22, 20], F32)]
_SETS = [
    ("437-477", "404-441", _NULLS_EQ, 0, 0, {1: ([1, 3, 0, 4, 6], [None, 19, 20, 21, 22]), 2: ([2, 5, 0, 4, 6], [None, 19, 20, 21, 22]),
                                            3: ([0, 4, 6], [20, 21, 22])}, I32),
    ("479-519", "443-480", _NULLS_NE, 1, 0, {1: ([0, 1, 2, 3, 4, 6], [20, None, None, 19, 21, 22]),
                                            2: ([1, 2, 4, 5, 6, 7], [None, None, 21, 19, 22, 20]), 3: ([1, 2, 4, 6], [None, None, 21, 22])}, I32),
    ("521-561", "482-519", _NANS_EQ, 0, 0, {1: ([0, 1, 3, 4, 6], [20.0, NAN, 19, 21, 22]), 2: ([0, 2, 4, 5, 6], [20.0, NAN, 21, 19, 22]),
                                           3: ([0, 4, 6], [20.0, 21, 22])}, F32),
    ("563-603", "521-558", _NANS_NE, 0, 1, {1: ([0, 1, 2, 3, 4, 6], [20.0, NAN, NAN, 19, 21, 22]),
                                           2: ([1, 2, 4, 5, 6, 7], [NAN, NAN, 21, 19, 22, 20]), 3: ([1, 2, 4, 6], [NAN, NAN, 21, 22])}, F32),
]
for _dl, _sl, _tab, _ne, _nan, _exp, _kt in _SETS:
    for _keep, (_rows, _keys) in _exp.items():
        _stable = sorted(zip(_rows, _keys), key=lambda rk: rk[0])
        _e = [([r for r, _ in _stable], I32), ([k for _, k in _stable], _kt)]
        CASES.append(dict(src=f"distinct_tests.cpp:{_dl} keep={_keep}", op="distinct", table=_tab, keys=[1], keep=_keep,
                          nulls_equal=_ne, nans_equal=_nan, expected=_e))
        CASES.append(dict(src=f"stable_distinct_tests.cpp:{_sl} keep={_keep}", op="stable_distinct", table=_tab, keys=[1], keep=_keep,
                          nulls_equal=_ne, nans_equal=_nan, expected=_e))
