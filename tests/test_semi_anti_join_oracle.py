"""CPU: the left semi / anti join oracle (tests/semi_anti_oracle.py) against the reference's known answers
(tests/golden/semi_anti_join_cases.py) and the row-equality rules the device path follows."""
import numpy as np
import pytest

from tests import semi_anti_oracle as osa
from tests.golden.semi_anti_join_cases import CASES
from tests.helpers import make_col


def case_cols(spec):
    return [make_col(vals, dt) for vals, dt in spec]


@pytest.mark.parametrize("case", CASES, ids=[c["src"] for c in CASES])
def test_oracle_golden(case):
    left, right = case_cols(case["left"]), case_cols(case["right"])
    assert osa.left_semi_join(left, right, case["nulls_equal"]).tolist() == case["semi"]
    assert osa.left_anti_join(left, right, case["nulls_equal"]).tolist() == case["anti"]


def test_oracle_row_equality():
    nan_a = np.frombuffer(np.array([0x7FF8000000000001], np.uint64).tobytes(), np.float64)[0]
    nan_b = np.frombuffer(np.array([0xFFF0000000000002], np.uint64).tobytes(), np.float64)[0]
    left = [make_col([nan_a, -0.0, 0.0, np.inf, -np.inf, 1.5, None], "float64")]
    right = [make_col([nan_b, 0.0, -np.inf, None], "float64")]
    assert osa.left_semi_join(left, right, osa.EQUAL).tolist() == [0, 1, 2, 4, 6]
    assert osa.left_semi_join(left, right, osa.UNEQUAL).tolist() == [0, 1, 2, 4]
    assert osa.left_anti_join(left, right, osa.UNEQUAL).tolist() == [3, 5, 6]
    # multi-column: every column equal, null == null only under EQUAL
    l2 = [make_col([1, 1, None, 2], "int64"), make_col([5, 6, 7, None], "int16")]
    r2 = [make_col([1, None, 2], "int64"), make_col([6, 7, None], "int16")]
    assert osa.left_semi_join(l2, r2, osa.EQUAL).tolist() == [1, 2, 3]
    assert osa.left_semi_join(l2, r2, osa.UNEQUAL).tolist() == [1]


def test_oracle_errors_after_early_returns():
    a = [make_col([1, 2], "int32")]
    with pytest.raises(ValueError):
        osa.left_semi_join(a, [make_col([1], "int64")])
    with pytest.raises(ValueError):
        osa.left_anti_join(a, a + a)
    # an empty side returns before any shape check
    assert osa.left_anti_join(a, []).tolist() == [0, 1]
    assert osa.left_semi_join([], a + a).tolist() == []
