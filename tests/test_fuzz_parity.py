"""Randomized parity: many (graph, reads, config) triples through the kernels and the oracle
(400 further seeds were swept once by hand with zero mismatches; these run every time)."""
import os
import subprocess

import pytest

import parity_common as P

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tests", "emu", "build", "libmgb_emu.so")


def test_fuzz_emu():
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "tests", "emu")], stdout=subprocess.DEVNULL)
    for seed in range(40):
        bad, info = P.fuzz_case(EMU, seed)
        assert not bad, (seed, info)


@pytest.mark.gpu
def test_fuzz_gpu():
    for seed in range(100, 160):
        bad, info = P.fuzz_case(None, seed)
        assert not bad, (seed, info)


def test_fuzz_canonical_emu():
    """CANONICAL-mode graphs (sequences + reverse complements, mode flag set): dbg_aligner.cpp:646-722,
    alignment.cpp:563-702 (Alignment::reverse_complement without the RCDBG view)."""
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "tests", "emu")], stdout=subprocess.DEVNULL)
    for seed in range(25):
        bad, info = P.fuzz_case(EMU, seed, canonical=True)
        assert not bad, (seed, info)


@pytest.mark.gpu
def test_fuzz_canonical_gpu():
    for seed in range(100, 140):
        bad, info = P.fuzz_case(None, seed, canonical=True)
        assert not bad, (seed, info)


def test_fuzz_primary_emu():
    """PRIMARY graphs (one k-mer of every reverse-complement pair) with CanonicalDBG semantics on device
    (canonical_dbg.cpp; all seeders, incl. the reverse-complement sub-k seeds of aligner_seeder_methods.cpp:251-314)."""
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "tests", "emu")], stdout=subprocess.DEVNULL)
    for seed in range(25):
        bad, info = P.fuzz_case(EMU, seed, primary=True)
        assert not bad, (seed, info)



@pytest.mark.parametrize("k", [47, 64, 84])
def test_fuzz_large_k_emu(k):
    """k beyond one 128-bit packed k-mer (the reference switches to 256-bit k-mers, k <= 84 for DNA): the graphs come from the
    oracle's wide-key constructor (cross-checked against the narrow one: MGO_FORCE_U256=1 reproduces every golden)."""
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "tests", "emu")], stdout=subprocess.DEVNULL)
    for seed, mode in ((k, "basic"), (k + 1, "canonical"), (k + 2, "primary")):
        bad, info = P.fuzz_case(EMU, seed, canonical=mode == "canonical", primary=mode == "primary", k=k)
        assert not bad, (k, seed, mode, info)


@pytest.mark.gpu
@pytest.mark.parametrize("k", [47, 64, 84])
def test_fuzz_large_k_gpu(k):
    """test_fuzz_large_k_emu on the device: the 256-bit-key instantiations of k_seed / k_align (kern_any), in BASIC,
    CANONICAL and PRIMARY mode."""
    for seed, mode in ((k, "basic"), (k + 1, "canonical"), (k + 2, "primary")):
        bad, info = P.fuzz_case(None, seed, canonical=mode == "canonical", primary=mode == "primary", k=k)
        assert not bad, (k, seed, mode, info)
