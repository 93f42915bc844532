"""Score edges on the host emulation (tests/score_edges_common.py): random full DNA matrices in every graph mode, random
protein matrices through the alphabet-generic layout, the whole-read gates under per-letter diagonals, and the
configurations at the bound of check_config_scores."""
import os
import subprocess

import pytest

import score_edges_common as SE

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tests", "emu", "build", "libmgb_emu.so")


@pytest.fixture(scope="module", autouse=True)
def _emu_built():
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "tests", "emu")], stdout=subprocess.DEVNULL)


@pytest.mark.parametrize("mode", [0, 1, 2], ids=["basic", "canonical", "primary"])
def test_dna_matrix_fuzz_emu(mode):
    out = SE.dna_matrix_family(EMU, range(30), mode)
    assert None in out                       # some configurations are rejected: MGB_ERR_BAD_CONFIG == the oracle's ctor


def test_protein_matrix_fuzz_emu():
    out = [SE.protein_case(EMU, s) for s in range(25)]
    assert sum(o is not None for o in out) >= 15


@pytest.mark.parametrize("which", ["min_path_score", "min_cell_score"])
@pytest.mark.parametrize("diag", range(len(SE.WHOLE_READ_DIAGS)))
def test_whole_read_gates_per_letter_diag_emu(which, diag):
    """the host emulation has no path layout, so exact_path_strand is reached on the device only (test_score_edges_gpu)"""
    every, rc = SE.whole_read_gate_case(EMU, 400 + diag, SE.WHOLE_READ_DIAGS[diag], which)
    assert every >= 10 and rc > 0, (every, rc)


@pytest.mark.parametrize("name", SE.BOUND_PINNED + SE.BOUND_UNPINNED)
def test_config_bound_emu(name):
    assert SE.bound_case(EMU, name) == (name in SE.BOUND_PINNED)
    SE.bound_case(EMU, name, "insertions")


@pytest.mark.parametrize("exact_seeder", [False, True], ids=["mem", "exact"])
@pytest.mark.parametrize("mode", [0, 1], ids=["basic", "canonical"])
def test_shortcut_gate_snp_emu(mode, exact_seeder):
    SE.shortcut_gate_snp_case(EMU, mode, exact_seeder)


def test_text_route_score_edges_emu():
    """a subset of the families through mgb_align_batch_text, TSV and JSON == the host mirror"""
    SE.dna_matrix_family(EMU, range(8), 0, text=True)
    for s in range(4):
        SE.protein_case(EMU, s, text=True)
    SE.whole_read_gate_case(EMU, 400, SE.WHOLE_READ_DIAGS[0], "min_path_score", text=True)
    for name in SE.BOUND_PINNED + SE.BOUND_UNPINNED:
        SE.bound_case(EMU, name, text=True)
