"""Long reads with errors on the device (tests/long_reads_common.py): reads of 0.5 - 30 kbp against the oracle. On the
device the DP columns of thousands of query positions are spread over 32 lanes, conv_grow moves table entries with a
lane-strided copy, and the backtrack writes CIGARs and node paths thousands of entries long. Each input must reach the
align pass it reaches on the emulation, and every retry pass must allocate arenas only for the reads it holds: a
single 30 kbp read retried at scale 64 needs one arena of about 24 GB, where four would not fit on an 80 GB card."""
import pytest

import long_reads_common as LR
import text_common as T

pytestmark = pytest.mark.gpu
LIB = None   # product library (metagraph_b200/_lib/libmgb.so)


def _check_grids(name, run):
    """one grid line per pass; no more arenas than warps; after pass 0 no more arenas than reads retried"""
    assert len(run.grids) == run.passes, (name, run.grids)
    n_reads = len(LR.LongReads(name).inp.reads)
    for p, (warps, _, stride, arenas) in enumerate(run.grids):
        assert 1 <= arenas <= min(warps, n_reads if p == 0 else run.stats["num_reads_retried"]), (name, p, run.grids)
    if name.startswith("single"):
        assert all(g[3] == 1 for g in run.grids), (name, run.grids)


@pytest.mark.parametrize("name,cfg", sorted(LR.PASSES), ids=["%s-%s" % nc for nc in sorted(LR.PASSES)])
def test_long_reads_gpu(name, cfg, monkeypatch, capfd):
    run = LR.check(LIB, name, cfg, trace=(monkeypatch, capfd))
    assert (run.stats["num_reads_retried"] > 0) == (LR.PASSES[(name, cfg)] > 1), (name, cfg, run.stats)
    assert run.passes == LR.PASSES[(name, cfg)], (name, cfg, run.passes, run.grids)
    _check_grids(name, run)


def test_long_reads_counters_gpu():
    """the exact-path shortcut off: the five DP counters == the oracle's"""
    LR.check(LIB, "lengths", "x27", shortcut=False)


def test_mixed_one_block_gpu(monkeypatch, capfd):
    """k_align's four warps of a single block align all 2 508 reads of the mixed batch, one after another"""
    monkeypatch.setenv("MGB_TEST_MAX_BLOCKS", "1")
    run = LR.check(LIB, "mixed", "x27", trace=(monkeypatch, capfd))
    assert run.passes == LR.PASSES[("mixed", "x27")], run.passes
    assert all(g[0] == 4 for g in run.grids), run.grids
    _check_grids("mixed", run)


@pytest.mark.parametrize("name", ["lengths", "mixed"])
def test_long_reads_text_gpu(name):
    """mgb_align_batch_text in TSV and JSON == the host mirror over mgb_align_batch's records"""
    lr = LR.LongReads(name)
    idx = lr.index(LIB)
    try:
        _, recs, st = T.check_text(idx, lr.cfg("x27"), lr.inp.reads)
    finally:
        idx.close()
    assert st["num_reads_retried"] > 0
    assert sum(1 for p in recs if p) >= len(recs) // 2
