"""Long reads with errors on the host emulation (tests/long_reads_common.py): reads of 0.5 - 30 kbp against the oracle,
with the reach of each input: reads retried with larger arenas, the number of align passes, convergence-table entries
moved to new segments, and in the mixed batch the 150 bp reads that are not staged on chip because the batch holds
a read over 511 bp. test_long_reads_gpu.py runs the same inputs on the device and expects the same passes."""
import os
import subprocess

import pytest

import long_reads_common as LR

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tests", "emu", "build", "libmgb_emu.so")


@pytest.fixture(scope="module", autouse=True)
def _emu_built():
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "tests", "emu")], stdout=subprocess.DEVNULL)


@pytest.mark.parametrize("name,cfg", sorted(LR.PASSES), ids=["%s-%s" % nc for nc in sorted(LR.PASSES)])
def test_long_reads_emu(name, cfg, monkeypatch, capfd):
    run = LR.check(EMU, name, cfg, trace=(monkeypatch, capfd))
    assert (run.stats["num_reads_retried"] > 0) == (LR.PASSES[(name, cfg)] > 1), (name, cfg, run.stats)
    assert run.passes == LR.PASSES[(name, cfg)], (name, cfg, run.passes)
    assert run.hits["read_overflow"] == run.stats["num_reads_retried"], run.hits
    assert run.hits["conv_move"] > 0, run.hits
    if name == "mixed":
        # one read over 511 bp: no read of the batch is staged on chip, the 2 500 short ones included
        assert run.hits["unstaged_read"] >= len(LR.LongReads(name).inp.reads), run.hits


def test_long_reads_counters_emu():
    """the exact-path shortcut off: the five DP counters == the oracle's"""
    LR.check(EMU, "lengths", "x27", shortcut=False)
