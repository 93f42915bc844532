"""The host emulation and the oracle built with UndefinedBehaviorSanitizer, run on a subset of the score-edge families
(tests/score_edges_common.py) in a subprocess: no `runtime error:` from the kernel sources. Past the range the
reference keeps its scores in (DESIGN.md §5) the kernels wrap on purpose, with explicit modulo-2^32 adds."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
UBSAN = "-fsanitize=undefined -fno-sanitize=alignment,vptr -fsanitize=float-cast-overflow"
EMU = os.path.join(ROOT, "tests", "emu", "build", "libmgb_emu_ubsan.so")
ORACLE = os.path.join(ROOT, "oracle", "build", "libmgo_ubsan.so")

SCRIPT = r"""
import sys
sys.path.insert(0, %(root)r); sys.path.insert(0, %(tests)r)
import oracle_lib
oracle_lib.LIB = %(oracle)r
import score_edges_common as SE
lib = %(emu)r
for mode in (0, 1, 2):
    SE.dna_matrix_family(lib, range(6), mode)
for s in range(6):
    SE.protein_case(lib, s)
SE.whole_read_gate_case(lib, 400, SE.WHOLE_READ_DIAGS[0], "min_path_score")
for name in SE.BOUND_PINNED + SE.BOUND_UNPINNED:
    SE.bound_case(lib, name)
print("score edges done")
"""


@pytest.fixture(scope="module")
def ubsan_libs():
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "tests", "emu"), "OUT=build/libmgb_emu_ubsan.so",
                           "CXX=g++ " + UBSAN], stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL)
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "oracle"), "OUT=build/libmgo_ubsan.so",
                           "CXXFLAGS=-O1 -g -std=c++17 -fPIC " + UBSAN], stdout=subprocess.DEVNULL,
                          stderr=subprocess.DEVNULL)
    return EMU, ORACLE


def test_score_edges_ubsan(ubsan_libs):
    emu, oracle = ubsan_libs
    code = SCRIPT % dict(root=ROOT, tests=os.path.join(ROOT, "tests"), oracle=oracle, emu=emu)
    env = dict(os.environ, UBSAN_OPTIONS="print_stacktrace=0:halt_on_error=0")
    r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0 and "score edges done" in r.stdout, r.stderr[-3000:]
    kernel = [l for l in r.stderr.splitlines() if "runtime error:" in l and "metagraph_b200/csrc/" in l]
    assert not kernel, "\n".join(sorted(set(kernel))[:20])
