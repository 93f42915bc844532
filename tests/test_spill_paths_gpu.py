"""k_align's spill, migration and retry paths on the device. When a read outgrows the aligner's on-chip working set,
its DP columns move to arena scratch (created there, or moved mid-column), its best-first queue and next-nodes list
migrate to the arena, its query strands stay in global memory, or it overflows its arena and is retried with a larger
one. Those moves are warp-cooperative copies, so a race between lanes can only show on the GPU. The pressure inputs
(parity_common.PRESSURE_INPUTS; the emulation tests show that each reaches its path) run here under every knob that
moves an on-chip limit or switches a path off: each run must equal the oracle line for line, node paths included, and
the default run's DP counters."""
import pytest

import parity_common as P

pytestmark = pytest.mark.gpu
LIB = None   # product library (metagraph_b200/_lib/libmgb.so)


@pytest.mark.parametrize("name", P.PRESSURE_INPUTS)
def test_spill_knobs_gpu(name, monkeypatch):
    runs = P.pressure_knob_matrix(LIB, name, monkeypatch)
    if name == "retry":
        # some reads overflow their arena at scale 1, also when the batch runs as three pieces (several heaps merged)
        for knob in ("default", "pieces3"):
            assert 0 < runs[knob][0]["num_reads_retried"] < len(P.pressure_input(name)[2]), (knob, runs[knob][0])
