"""Score edges on the device (tests/score_edges_common.py): random full DNA matrices in every graph mode, also under the
spill knobs that move scoring to each of its sites (chain loop with the packed profile, general path, alphabet-generic
layout, reads not staged on chip), random protein matrices through kern_any, the whole-read gates under per-letter
diagonals with k_prepare_exact answering reads, and the configurations at the bound of check_config_scores."""
import re

import pytest

import parity_common as P
import score_edges_common as SE

LIB = None
KNOBS = [kv for kv in P.SPILL_KNOBS if kv[0] in ("default", "nofast", "wide", "lq0")]


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [0, 1, 2], ids=["basic", "canonical", "primary"])
def test_dna_matrix_fuzz_gpu(mode):
    out = SE.dna_matrix_family(LIB, range(100, 160), mode)
    assert None in out                       # some configurations are rejected: MGB_ERR_BAD_CONFIG == the oracle's ctor


@pytest.mark.gpu
@pytest.mark.parametrize("knob", KNOBS, ids=[k for k, _ in KNOBS])
def test_dna_matrix_knobs_gpu(knob, monkeypatch):
    for var, val in knob[1].items():
        monkeypatch.setenv(var, val)
    for mode in ((0,) if knob[0] == "wide" else (0, 1, 2)):     # CANONICAL / PRIMARY run on the DNA block layout only
        SE.dna_matrix_family(LIB, range(200, 212), mode)


@pytest.mark.gpu
def test_protein_matrix_fuzz_gpu():
    out = [SE.protein_case(LIB, s) for s in range(100, 150)]
    assert sum(o is not None for o in out) >= 30


@pytest.mark.gpu
@pytest.mark.parametrize("which", ["min_path_score", "min_cell_score"])
@pytest.mark.parametrize("diag", range(len(SE.WHOLE_READ_DIAGS)))
def test_whole_read_gates_per_letter_diag_gpu(which, diag, monkeypatch, capfd):
    monkeypatch.setenv("MGB_DEBUG", "1")
    """k_prepare_exact answers reads (exact_path_strand), also in the run of reverse-complement reads alone, the last
    call of the case"""
    SE.whole_read_gate_case(LIB, 400 + diag, SE.WHOLE_READ_DIAGS[diag], which)
    err = capfd.readouterr().err
    answered = [int(x) for x in re.findall(r"k_prepare_exact answered (\d+)", err)]
    assert answered and answered[-1] > 0, err[-2000:]


@pytest.mark.gpu
@pytest.mark.parametrize("name", SE.BOUND_PINNED + SE.BOUND_UNPINNED)
def test_config_bound_gpu(name):
    assert SE.bound_case(LIB, name) == (name in SE.BOUND_PINNED)
    SE.bound_case(LIB, name, "insertions")


@pytest.mark.gpu
@pytest.mark.parametrize("exact_seeder", [False, True], ids=["mem", "exact"])
@pytest.mark.parametrize("mode", [0, 1], ids=["basic", "canonical"])
def test_shortcut_gate_snp_gpu(mode, exact_seeder):
    SE.shortcut_gate_snp_case(LIB, mode, exact_seeder)


@pytest.mark.gpu
def test_text_route_score_edges_gpu():
    """a subset of the families through mgb_align_batch_text, TSV and JSON == the host mirror"""
    for mode in (0, 1, 2):
        SE.dna_matrix_family(LIB, range(100, 110), mode, text=True)
    for s in range(100, 106):
        SE.protein_case(LIB, s, text=True)
    SE.whole_read_gate_case(LIB, 400, SE.WHOLE_READ_DIAGS[0], "min_path_score", text=True)
    for name in SE.BOUND_PINNED + SE.BOUND_UNPINNED:
        SE.bound_case(LIB, name, text=True)
