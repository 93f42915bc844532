"""The extender's stop rules on the host emulation: RAM and node budgets chosen from the oracle's trace of its own stop
tests, no_backtrack, and the whole-read and exact-path shortcuts at budgets that stop any search; lines and DP counters
equal the oracle's (tests/budget_common.py). The emulation counts the four stop sites, which shows each is reached.
test_budgets_gpu.py runs the same matrix on the device."""
import os
import subprocess

import pytest

import budget_common as B

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tests", "emu", "build", "libmgb_emu.so")
STOPS = ("ram_stop_general", "nodes_stop_general", "ram_stop_chain", "nodes_stop_chain")


@pytest.fixture(scope="module", autouse=True)
def _emu_built():
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "tests", "emu")], stdout=subprocess.DEVNULL)


@pytest.mark.parametrize("name", B.BUDGET_INPUTS)
def test_budget_matrix_emu(name):
    assert B.budget_matrix(EMU, name) > 0


@pytest.mark.parametrize("name", B.BUDGET_INPUTS)
def test_no_backtrack_emu(name):
    B.no_backtrack_case(EMU, name)


def test_shortcuts_at_extreme_budgets_emu():
    B.shortcut_budget_cases(EMU)


def test_stop_sites_reached_emu():
    """each copy of each stop test ends searches: the general loop's and chain_loop's RAM and node exits"""
    hits = B.stop_site_hits(EMU)
    assert all(hits[s] > 0 for s in STOPS), hits


def test_stop_sites_without_register_path_emu(monkeypatch):
    """without the register path every column is a general one: only the general loop's copies stop searches"""
    monkeypatch.setenv("MGB_TEST_NOFAST", "1")
    hits = B.stop_site_hits(EMU)
    assert hits["ram_stop_general"] > 0 and hits["nodes_stop_general"] > 0, hits
    assert hits["ram_stop_chain"] == 0 and hits["nodes_stop_chain"] == 0, hits
