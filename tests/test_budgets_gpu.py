"""The extender's stop rules on the device (tests/budget_common.py): RAM and node budgets chosen from the oracle's
trace of its own stop tests, no_backtrack, and the shortcuts at budgets that stop any search. On the device the
general loop scans a column with 32 lanes and reductions and chain_loop keeps several cells per lane; both must stop
where the reference stops, which the DP counters show column for column."""
import pytest

import budget_common as B
import parity_common as P

pytestmark = pytest.mark.gpu
LIB = None   # product library (metagraph_b200/_lib/libmgb.so)


@pytest.mark.parametrize("name", B.BUDGET_INPUTS)
def test_budget_matrix_gpu(name):
    assert B.budget_matrix(LIB, name) > 0


@pytest.mark.parametrize("name", B.BUDGET_INPUTS)
def test_no_backtrack_gpu(name):
    B.no_backtrack_case(LIB, name)


def test_shortcuts_at_extreme_budgets_gpu():
    B.shortcut_budget_cases(LIB)


@pytest.mark.parametrize("name", B.PRESSURE_BUDGET_INPUTS)
def test_budget_knobs_gpu(name, monkeypatch):
    B.budget_knob_matrix(LIB, name, monkeypatch)


@pytest.mark.parametrize("case", P.RANDOM_CASES, ids=[str(c[0]) for c in P.RANDOM_CASES])
def test_random_counters_gpu(case):
    """the shortcut off: the kernel's five DP counters == the oracle's, so any change to what the search explores
    shows even when the answer stays the same"""
    B.random_counters_case(LIB, case)
