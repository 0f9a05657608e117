"""Known answers of the reference's replacement tests for the fixed-width types, transcribed with their data and names from
cpp/tests/replace/{replace_nulls_tests,replace_nans_tests,replace_tests,clamp_test,normalize_replace_tests}.cpp.

Each case runs over `types` (the typed tests' NumericTypes without BOOL8, or FLOAT32 / FLOAT64; a plain TEST_F keeps its own
type). Arguments are col(values, valid, type) or scl(value, valid, type), type None meaning the case's type. `expect` holds the
values and `expect_valid` their validity (None: all valid), compared at valid rows as CUDF_TEST_EXPECT_COLUMNS_EQUAL does,
bit for bit where `bitwise` is set; `raises` is TypeError for cudf::data_type_error and RuntimeError for cudf::logic_error."""
INT8, INT16, INT32, INT64, UINT8, UINT16, UINT32, UINT64, FLOAT32, FLOAT64 = 1, 2, 3, 4, 5, 6, 7, 8, 9, 10
NUMERIC = [INT8, INT16, INT32, INT64, UINT8, UINT16, UINT32, UINT64, FLOAT32, FLOAT64]
FLOATS = [FLOAT32, FLOAT64]
NAN = float("nan")
PRECEDING, FOLLOWING = 0, 1


def col(values, valid=None, type=None):
    return {"col": list(values), "valid": valid, "type": type}


def scl(value, valid=True, type=None):
    return {"scalar": value, "valid": valid, "type": type}


def case(src, fn, args, types, expect=None, expect_valid=None, raises=None, bitwise=False):
    return dict(src=src, fn=fn, args=args, types=types, expect=expect, expect_valid=expect_valid, raises=raises, bitwise=bitwise)


V5 = [0, 0, 0, 0, 0, 1, 1, 1, 1, 1]
NANS10 = [NAN, 1.0, NAN, 3.0, 4.0, NAN, NAN, 7.0, 8.0, 9.0]

CASES = [
    # ---- replace_nulls_tests.cpp --------------------------------------------------------------------------------------
    case("replace_nulls_tests.cpp:45 ReplaceErrorTest.SizeMismatch", "replace_nulls",
         [col([7, 5, 6, 3, 1, 2, 8, 4], [0, 0, 1, 1, 1, 1, 1, 1]), col([10, 11, 12, 13])], [INT32], raises="RuntimeError"),
    case("replace_nulls_tests.cpp:55 ReplaceErrorTest.TypeMismatch", "replace_nulls",
         [col([7, 5, 6, 3, 1, 2, 8, 4], [0, 0, 1, 1, 1, 1, 1, 1]), col([10, 11, 12, 13, 14, 15, 16, 17], type=FLOAT32)], [INT32],
         raises="TypeError"),
    case("replace_nulls_tests.cpp:66 ReplaceErrorTest.TypeMismatchScalar", "replace_nulls",
         [col([7, 5, 6, 3, 1, 2, 8, 4], [0, 0, 1, 1, 1, 1, 1, 1]), scl(1, type=FLOAT32)], [INT32], raises="TypeError"),
    case("replace_nulls_tests.cpp:267 ReplaceNullsTest.ReplaceColumn", "replace_nulls",
         [col(range(10), V5), col(range(10))], NUMERIC, expect=list(range(10))),
    case("replace_nulls_tests.cpp:284 ReplaceNullsTest.ReplaceColumn_Empty", "replace_nulls", [col([]), col([])], NUMERIC,
         expect=[]),
    case("replace_nulls_tests.cpp:291 ReplaceNullsTest.ReplaceScalar", "replace_nulls", [col(range(10), V5), scl(1)], NUMERIC,
         expect=[1, 1, 1, 1, 1, 5, 6, 7, 8, 9]),
    case("replace_nulls_tests.cpp:308 ReplaceNullsTest.ReplacementHasNulls", "replace_nulls",
         [col([7, 5, 6, 3, 1, 2, 8, 4], [0, 0, 1, 1, 1, 1, 1, 1]), col([4, 5, 6, 7, 8, 9, 0, 1], [1, 0, 1, 1, 1, 1, 1, 1])], NUMERIC,
         expect=[4, 5, 6, 3, 1, 2, 8, 4], expect_valid=[1, 0, 1, 1, 1, 1, 1, 1]),
    case("replace_nulls_tests.cpp:385 ReplaceNullsPolicyTest.PrecedingFill", "replace_nulls",
         [col([42, 2, 1, -10, 20, -30], [1, 0, 0, 1, 0, 1]), PRECEDING], NUMERIC, expect=[42, 42, 42, -10, -10, -30]),
    case("replace_nulls_tests.cpp:399 ReplaceNullsPolicyTest.FollowingFill", "replace_nulls",
         [col([42, 2, 1, -10, 20, -30], [1, 0, 0, 1, 0, 1]), FOLLOWING], NUMERIC, expect=[42, -10, -10, -10, -30, -30]),
    case("replace_nulls_tests.cpp:413 ReplaceNullsPolicyTest.PrecedingFillLeadingNulls", "replace_nulls",
         [col([1, 2, 3, 4, 5], [0, 0, 1, 0, 1]), PRECEDING], NUMERIC, expect=[1, 2, 3, 3, 5], expect_valid=[0, 0, 1, 1, 1]),
    case("replace_nulls_tests.cpp:427 ReplaceNullsPolicyTest.FollowingFillTrailingNulls", "replace_nulls",
         [col([1, 2, 3, 4, 5], [1, 0, 1, 0, 0]), FOLLOWING], NUMERIC, expect=[1, 3, 3, 4, 5], expect_valid=[1, 1, 1, 0, 0]),
    # ---- replace_nans_tests.cpp ---------------------------------------------------------------------------------------
    case("replace_nans_tests.cpp:18 ReplaceNaNsErrorTest.SizeMismatch", "replace_nans",
         [col([7, 5, 6, 3, 1, 8, 4]), col([10, 11, 12, 13])], [FLOAT32], raises="RuntimeError"),
    case("replace_nans_tests.cpp:27 ReplaceNaNsErrorTest.TypeMismatch", "replace_nans",
         [col([7, 5, 6, 3, 1, 2, 8, 4]), col([10, 11, 12, 13, 14, 15, 16, 17], type=FLOAT64)], [FLOAT32], raises="RuntimeError"),
    case("replace_nans_tests.cpp:36 ReplaceNaNsErrorTest.TypeMismatchScalar", "replace_nans",
         [col([7, 5, 6, 3, 1, 2, 8, 4]), scl(1, type=FLOAT32)], [FLOAT64], raises="RuntimeError"),
    case("replace_nans_tests.cpp:45 ReplaceNaNsErrorTest.NonFloatType", "replace_nans",
         [col([7, 5, 6, 3, 1, 2, 8, 4]), scl(1, type=FLOAT32)], [INT32], raises="RuntimeError"),
    case("replace_nans_tests.cpp:80 ReplaceNaNsTest.ReplaceColumn", "replace_nans", [col(NANS10), col(range(10))], FLOATS,
         expect=list(range(10))),
    case("replace_nans_tests.cpp:96 ReplaceNaNsTest.ReplaceColumnNullable", "replace_nans", [col(NANS10, V5), col(range(10))],
         FLOATS, expect=list(range(10)), expect_valid=V5),
    case("replace_nans_tests.cpp:116 ReplaceNaNsTest.ReplacementHasNulls", "replace_nans",
         [col([7.0, NAN, 6.0, 3.0, NAN, 2.0, 8.0, 4.0]), col([4, 5, 6, 7, 8, 9, 0, 1], [1, 0, 1, 1, 1, 1, 1, 1])], FLOATS,
         expect=[7.0, 5.0, 6.0, 3.0, 8.0, 2.0, 8.0, 4.0], expect_valid=[1, 0, 1, 1, 1, 1, 1, 1]),
    case("replace_nans_tests.cpp:138 ReplaceNaNsTest.ReplaceColumn_Empty", "replace_nans", [col([]), col([])], FLOATS, expect=[]),
    case("replace_nans_tests.cpp:145 ReplaceNaNsTest.ReplaceScalar", "replace_nans", [col(NANS10, V5), scl(1)], FLOATS,
         expect=[0, 1, 2, 3, 4, 1, 1, 7, 8, 9], expect_valid=V5),
    case("replace_nans_tests.cpp:164 ReplaceNaNsTest.ReplaceNullScalar", "replace_nans", [col(NANS10, V5), scl(1, valid=False)],
         FLOATS, expect=[0, 1, 2, 3, 4, 1, 1, 7, 8, 9], expect_valid=[0, 0, 0, 0, 0, 0, 0, 1, 1, 1]),
    # ---- replace_tests.cpp (find_and_replace_all) -----------------------------------------------------------------------
    case("replace_tests.cpp:49 ReplaceErrorTest.SizeMismatch", "find_and_replace_all",
         [col([7, 5, 6, 3, 1, 2, 8, 4]), col([10, 11, 12, 13]), col([15, 16, 17])], [INT32], raises="RuntimeError"),
    case("replace_tests.cpp:61 ReplaceErrorTest.TypeMismatch", "find_and_replace_all",
         [col([7, 5, 6, 3, 1, 2, 8, 4]), col([10, 11, 12], type=FLOAT32), col([15, 16, 17])], [INT32], raises="TypeError"),
    case("replace_tests.cpp:73 ReplaceErrorTest.NullInOldValues", "find_and_replace_all",
         [col([7, 5, 6, 3, 1, 2, 8, 4]), col([10, 11, 12, 13], [0, 1, 0, 1]), col([15, 16, 17, 18])], [INT32], raises="RuntimeError"),
    case("replace_tests.cpp:397 ReplaceTest.ReplaceEvenPosition", "find_and_replace_all",
         [col([1, 2, 3, 4, 5, 6, 7, 8]), col([2, 6, 4, 8]), col([0, 4, 2, 6])], NUMERIC, expect=[1, 0, 3, 2, 5, 4, 7, 6]),
    case("replace_tests.cpp:408 ReplaceTest.Unordered", "find_and_replace_all",
         [col([7, 5, 6, 3, 1, 2, 8, 4]), col([2, 6, 4, 8]), col([0, 4, 2, 6])], NUMERIC, expect=[7, 5, 4, 3, 1, 0, 6, 2]),
    case("replace_tests.cpp:419 ReplaceTest.NothingToReplace", "find_and_replace_all",
         [col([7, 5, 6, 3, 1, 2, 8, 4]), col([10, 11, 12]), col([15, 16, 17])], NUMERIC, expect=[7, 5, 6, 3, 1, 2, 8, 4]),
    case("replace_tests.cpp:430 ReplaceTest.EmptyData", "find_and_replace_all", [col([]), col([10, 11, 12]), col([15, 16, 17])],
         NUMERIC, expect=[]),
    case("replace_tests.cpp:441 ReplaceTest.EmptyReplace", "find_and_replace_all", [col([7, 5, 6, 3, 1, 2, 8, 4]), col([]), col([])],
         NUMERIC, expect=[7, 5, 6, 3, 1, 2, 8, 4]),
    case("replace_tests.cpp:452 ReplaceTest.NullsInData", "find_and_replace_all",
         [col([7, 5, 6, 3, 1, 2, 8, 4], [1, 1, 1, 0, 0, 1, 1, 1]), col([2, 6, 4, 8]), col([0, 4, 2, 6])], NUMERIC,
         expect=[7, 5, 4, 3, 1, 0, 6, 2], expect_valid=[1, 1, 1, 0, 0, 1, 1, 1]),
    case("replace_tests.cpp:466 ReplaceTest.NullsInNewValues", "find_and_replace_all",
         [col([7, 5, 6, 3, 1, 2, 8, 4]), col([2, 6, 4, 8]), col([0, 4, 2, 6], [0, 1, 1, 1])], NUMERIC,
         expect=[7, 5, 4, 3, 1, 0, 6, 2], expect_valid=[1, 1, 1, 1, 1, 0, 1, 1]),
    case("replace_tests.cpp:483 ReplaceTest.NullsInBoth", "find_and_replace_all",
         [col([7, 5, 6, 3, 1, 2, 8, 4], [1, 1, 1, 0, 0, 1, 1, 1]), col([2, 6, 4, 8]), col([0, 4, 2, 6], [1, 1, 0, 1])], NUMERIC,
         expect=[7, 5, 4, 3, 1, 0, 6, 2], expect_valid=[1, 1, 1, 0, 0, 1, 1, 0]),
    # ---- clamp_test.cpp -----------------------------------------------------------------------------------------------
    case("clamp_test.cpp ClampErrorTest.MisMatchingScalarTypes", "clamp",
         [col([1, 2, 3, 4, 5, 6]), scl(0, type=INT32), scl(0, type=INT64)], [INT32], raises="TypeError"),
    case("clamp_test.cpp ClampErrorTest.MisMatchingInputAndScalarTypes", "clamp",
         [col([1, 2, 3, 4, 5, 6]), scl(0, type=INT32), scl(0, type=INT32)], [INT64], raises="TypeError"),
    case("clamp_test.cpp ClampErrorTest.MisMatchingReplaceScalarTypes", "clamp",
         [col([1, 2, 3, 4, 5, 6]), scl(0, type=INT32), scl(0, type=INT64), scl(0, type=INT32), scl(0, type=INT32)], [INT64],
         raises="TypeError"),
    case("clamp_test.cpp ClampErrorTest.InValidCase1", "clamp",
         [col([1, 2, 3, 4, 5, 6]), scl(0, type=INT32), scl(0, False, type=INT32), scl(0, type=INT32), scl(0, type=INT32)], [INT64],
         raises="RuntimeError"),
    case("clamp_test.cpp ClampErrorTest.InValidCase2", "clamp",
         [col([1, 2, 3, 4, 5, 6]), scl(0, type=INT32), scl(0, type=INT32), scl(0, type=INT32), scl(0, False, type=INT32)], [INT64],
         raises="RuntimeError"),
    case("clamp_test.cpp ClampEmptyCaseTest.BothScalarEmptyInvalid", "clamp",
         [col([1, 2, 3, 4, 5, 6]), scl(0, False, type=INT32), scl(0, False, type=INT32)], [INT32], expect=[1, 2, 3, 4, 5, 6]),
    case("clamp_test.cpp ClampEmptyCaseTest.EmptyInput", "clamp", [col([]), scl(0, type=INT32), scl(0, type=INT32)], [INT32],
         expect=[]),
    case("clamp_test.cpp ClampTestNumeric.WithNoNull", "clamp", [col(range(11)), scl(2), scl(2), scl(8), scl(8)], NUMERIC,
         expect=[2, 2, 2, 3, 4, 5, 6, 7, 8, 8, 8]),
    case("clamp_test.cpp ClampTestNumeric.LowerNull", "clamp", [col(range(11)), scl(2, False), scl(2, False), scl(8), scl(8)],
         NUMERIC, expect=[0, 1, 2, 3, 4, 5, 6, 7, 8, 8, 8]),
    case("clamp_test.cpp ClampTestNumeric.UpperNull", "clamp", [col(range(11)), scl(2), scl(2), scl(8, False), scl(8, False)],
         NUMERIC, expect=[2, 2, 2, 3, 4, 5, 6, 7, 8, 9, 10]),
    case("clamp_test.cpp ClampTestNumeric.InputNull", "clamp",
         [col(range(11), [0, 1, 0, 1, 0, 1, 0, 1, 0, 1, 0]), scl(2), scl(2), scl(8), scl(8)], NUMERIC,
         expect=[2, 2, 2, 3, 4, 5, 6, 7, 8, 8, 8], expect_valid=[0, 1, 0, 1, 0, 1, 0, 1, 0, 1, 0]),
    case("clamp_test.cpp ClampTestNumeric.InputNulliWithReplace", "clamp",
         [col(range(11), [0, 1, 0, 1, 0, 1, 0, 1, 0, 1, 0]), scl(2), scl(16), scl(8), scl(32)], NUMERIC,
         expect=[16, 16, 2, 3, 4, 5, 6, 7, 8, 32, 32], expect_valid=[0, 1, 0, 1, 0, 1, 0, 1, 0, 1, 0]),
    case("clamp_test.cpp:286 ClampFloatTest.WithNANandNoNull", "clamp",
         [col([8.0, 6.0, NAN, 3.0, 4.0, 5.0, 1.0, NAN, 2.0, 9.0]), scl(2.0), scl(2.0), scl(6.0), scl(6.0)], FLOATS,
         expect=[6.0, 6.0, NAN, 3.0, 4.0, 5.0, 2.0, NAN, 2.0, 6.0]),
    case("clamp_test.cpp:310 ClampFloatTest.WithNANandNull", "clamp",
         [col([8.0, 6.0, NAN, 3.0, 4.0, 5.0, 1.0, NAN, 2.0, 9.0], [1, 1, 1, 0, 1, 1, 1, 0, 1, 1]), scl(2.0), scl(2.0), scl(6.0),
          scl(6.0)], FLOATS, expect=[6.0, 6.0, NAN, 3.0, 4.0, 5.0, 2.0, NAN, 2.0, 6.0], expect_valid=[1, 1, 1, 0, 1, 1, 1, 0, 1, 1]),
    case("clamp_test.cpp:336 ClampFloatTest.SignOfAFloat", "clamp",
         [col([2.0, 0.0, NAN, 4.0, -0.5, -1.0, 1.0, NAN, 0.5, 9.0], [1, 1, 1, 0, 1, 1, 1, 0, 1, 1]), scl(0.0), scl(-1.0), scl(0.0),
          scl(1.0)], FLOATS, expect=[1.0, 0.0, NAN, 4.0, -1.0, -1.0, 1.0, NAN, 1.0, 1.0], expect_valid=[1, 1, 1, 0, 1, 1, 1, 0, 1, 1]),
    # ---- normalize_replace_tests.cpp: compared bit for bit (CUDF_TEST_EXPECT_EQUAL_BUFFERS) -------------------------------
    case("normalize_replace_tests.cpp:47 ReplaceTest.NormalizeNansAndZerosFloat", "normalize_nans_and_zeros",
         [col([32.5, -0.0, 111.0, -NAN, NAN, 1.0, 0.0, 54.3])], [FLOAT32], expect=[32.5, 0.0, 111.0, NAN, NAN, 1.0, 0.0, 54.3],
         bitwise=True),
    case("normalize_replace_tests.cpp:60 ReplaceTest.NormalizeNansAndZerosDouble", "normalize_nans_and_zeros",
         [col([32.5, -0.0, 111.0, -NAN, NAN, 1.0, 0.0, 54.3])], [FLOAT64], expect=[32.5, 0.0, 111.0, NAN, NAN, 1.0, 0.0, 54.3],
         bitwise=True),
]
