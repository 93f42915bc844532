"""The index selects the route of whole-read exact answers: answering them from the raw reads (exact_path_strand,
k_prepare_exact) needs the k-mer hash index and the path layout, which only the device builds. On the host emulation the
graph has neither, so no read takes that route and k_exact_reads (exact_read_strand) still answers the exact ones, ==
oracle. The route itself is checked on the device by test_prepare_exact_gpu.py."""
import ctypes
import os
import subprocess

import pytest

import parity_common as P
from metagraph_b200 import _lib
from metagraph_b200.config import cli_defaults

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tests", "emu", "build", "libmgb_emu.so")


@pytest.fixture(scope="module", autouse=True)
def _emu_built():
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "tests", "emu")], stdout=subprocess.DEVNULL)


def path_read_hits():
    return ctypes.c_ulonglong.in_dll(_lib.load_library(EMU), "mgb_emu_path_read_hits").value


@pytest.mark.parametrize("k", [31, 15])
def test_prepare_exact_needs_path_layout_emu(k):
    before = path_read_hits()
    hits = P.whole_read_case(EMU, 3100 + k, k, cli_defaults(k, min_seed_length=k, max_seed_length=k))
    assert hits >= 20
    assert path_read_hits() == before
