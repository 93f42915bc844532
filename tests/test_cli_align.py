"""`python -m metagraph_b200 align`: every flag gives the configuration cli_defaults builds from the same values, the
options the command does not implement exit non-zero, and the whole command (on the host emulation of the kernels)
prints the oracle's lines for the example graphs, from plain and gzip input, whatever -p and --batch-size say."""
import ctypes
import gzip
import os
import subprocess
import sys

import pytest

import fastx_common as F
import oracle_lib as O
from metagraph_b200 import cli
from metagraph_b200.aligner import BOSSTable
from metagraph_b200.config import SIZE_MAX, cli_defaults, dna_scoring_matrix

EX = os.path.join(F.GOLD, "example_graphs")
GRAPHS = [("test_DNA_graph.dbg", "test_DNA_query.fa", "dna"), ("test_Protein_graph.dbg", "test_Protein_query.fa", "protein")]


@pytest.fixture(scope="module", autouse=True)
def _emu_built():
    subprocess.check_call(["make", "-C", os.path.join(F.ROOT, "tests", "emu")], stdout=subprocess.DEVNULL)


def c_bytes(cfg):
    c = cfg.to_c()
    return bytes((ctypes.c_char * ctypes.sizeof(c)).from_buffer_copy(c))


def cfg_of(argv, k=31, alphabet="dna"):
    return cli.config_of(cli.parse_args(argv + ["-i", "g.dbg", "r.fa"]), k, alphabet)


FLAGS = [  # (arguments, the cli_defaults keywords they stand for)
    ([], {}),
    (["--align-only-forwards"], dict(forward_and_reverse_complement=False)),
    (["--align-no-seed-complexity-filter"], dict(seed_complexity_filter=False)),
    (["--align-match-score", "3", "--align-mm-transition-penalty", "1", "--align-mm-transversion-penalty", "4"],
     dict(score_matrix=dna_scoring_matrix(3, -1, -4))),
    (["--align-gap-open-penalty", "7", "--align-gap-extension-penalty", "1"],
     dict(gap_opening_penalty=-7, gap_extension_penalty=-1)),
    (["--align-end-bonus", "2"], dict(left_end_bonus=2, right_end_bonus=2)),
    (["--align-alternative-alignments", "4"], dict(num_alternative_paths=4)),
    (["--align-min-path-score", "30"], dict(min_path_score=30)),
    (["--align-xdrop", "50"], dict(xdrop=50)),
    (["--align-min-seed-length", "40"], dict(min_seed_length=31)),           # capped at k (cli/align.cpp:39-40)
    (["--align-min-seed-length", "15"], dict(min_seed_length=15)),
    (["--align-max-seed-length", "25"], dict(max_seed_length=25)),
    (["--align-max-num-seeds-per-locus", "7"], dict(max_num_seeds_per_locus=7)),
    (["--align-max-nodes-per-seq-char", "2.5"], dict(max_nodes_per_seq_char=2.5)),
    (["--align-min-exact-match", "0.0"], dict(min_exact_match=0.0)),
    (["--align-max-ram", "50"], dict(max_ram_per_alignment=50.0)),
    (["--align-rel-score-cutoff", "0.5"], dict(rel_score_cutoff=0.5)),
]


@pytest.mark.parametrize("i", range(len(FLAGS)))
def test_flag_config(i):
    argv, kw = FLAGS[i]
    exp = cli_defaults(31, **dict(dict(seed_complexity_filter=True), **kw))
    assert c_bytes(cfg_of(argv)) == c_bytes(exp)


def test_edit_distance_and_protein_config():
    # --align-edit-distance: unit costs and no end bonus, whatever --align-end-bonus says (aligner_config.cpp:128-148)
    assert c_bytes(cfg_of(["--align-edit-distance", "--align-end-bonus", "3"])) == \
        c_bytes(cli_defaults(31, edit_distance=True, seed_complexity_filter=True))
    assert c_bytes(cfg_of(["--align-match-score", "5"], 20, "protein")) == \
        c_bytes(cli_defaults(20, "protein", seed_complexity_filter=True))
    assert cfg_of([], 20, "protein").forward_and_reverse_complement is False
    assert cfg_of(["--align-max-seed-length", str(SIZE_MAX)]).max_seed_length == SIZE_MAX


@pytest.mark.parametrize("argv", [["--map"], ["-a", "x.annodbg"], ["--annotator", "x"], ["--align-chain"],
                                  ["--align-post-chain"], ["-o", "out.gfa"], ["--align-min-seed-length", "30",
                                  "--align-max-seed-length", "20"], ["--align-gap-open-penalty", "-1"],
                                  ["--align-alternative-alignments", "0"]])
def test_refused(argv, tmp_path):
    r = subprocess.run([sys.executable, "-m", "metagraph_b200", "align", "-i", os.path.join(EX, GRAPHS[0][0])] + argv
                       + [os.path.join(EX, GRAPHS[0][1])], cwd=F.ROOT, capture_output=True,
                       env=dict(os.environ, MGB_LIB=F.EMU, PYTHONPATH=F.ROOT))
    assert r.returncode != 0 and r.stderr


def run_command(args, lib=None):
    env = dict(os.environ, PYTHONPATH=F.ROOT)
    if lib:
        env["MGB_LIB"] = lib
    r = subprocess.run([sys.executable, "-m", "metagraph_b200", "align"] + args, cwd=F.ROOT, capture_output=True,
                       env=env)
    assert r.returncode == 0, r.stderr.decode()
    return r.stdout


def oracle_text(dbg, query, alphabet, argv=()):
    t = BOSSTable.from_dbg(os.path.join(EX, dbg), lib=F.EMU)
    cfg = cfg_of(list(argv), t.k, alphabet)
    names, reads = F.read_fasta(os.path.join(EX, query))
    g = O.OracleGraph(t.k, arrays=(t.W, t.last, t.F), alphabet=alphabet)
    lines = g.align_tsv(cfg, reads, headers=[n.decode() for n in names])
    return "".join(l + "\n" for l in lines).encode()


def command_case(tmp_path, lib):
    """the command on both example graphs against the oracle, from plain and .gz input, with -p / --batch-size and
    with -o"""
    for dbg, query, alphabet in GRAPHS:
        exp = oracle_text(dbg, query, alphabet)
        plain = os.path.join(EX, query)
        gz = str(tmp_path / (query + ".gz"))
        with gzip.open(gz, "wb") as f:
            f.write(open(plain, "rb").read())
        g = os.path.join(EX, dbg)
        assert run_command(["-i", g, plain], lib) == exp
        assert run_command(["-i", g, gz], lib) == exp
        assert run_command(["-i", g, "-p", "8", "--batch-size", "10", plain], lib) == exp
        out = str(tmp_path / "out.tsv")
        # -o is reopened for every input file: it holds the last file's output
        other = str(tmp_path / "one.fa")
        open(other, "wb").write(b">x\n" + F.read_fasta(plain)[1][0] + b"\n")
        assert run_command(["-i", g, "-o", out, other, plain], lib) == b""
        assert open(out, "rb").read() == exp


def test_command_emu(tmp_path):
    command_case(tmp_path, F.EMU)


def test_chunked_file_emu(tmp_path):
    """a file read in chunks smaller than its records gives the text of one chunk"""
    from metagraph_b200.aligner import B200Aligner, DBGSuccinctIndex
    t = BOSSTable.from_dbg(os.path.join(EX, GRAPHS[0][0]), lib=F.EMU)
    idx = DBGSuccinctIndex(t, lib=F.EMU)
    try:
        al = B200Aligner(idx, cli_defaults(t.k))
        path = os.path.join(F.GOLD, "transcripts_100.fa")
        import io
        whole, small = io.BytesIO(), io.BytesIO()
        cli.align_file(al, path, whole)
        cli.align_file(al, path, small, chunk_bytes=97)
        assert whole.getvalue() == small.getvalue() and whole.getvalue().count(b"\n") == 100
    finally:
        idx.close()


def test_file_growth_and_early_end_emu(tmp_path):
    """a record of many chunks is parsed a logarithmic number of times; a malformed record ends the file there"""
    import io
    from metagraph_b200.aligner import B200Aligner, DBGSuccinctIndex
    t = BOSSTable.from_dbg(os.path.join(EX, GRAPHS[0][0]), lib=F.EMU)
    idx = DBGSuccinctIndex(t, lib=F.EMU)
    try:
        al = B200Aligner(idx, cli_defaults(t.k))
        calls = []
        orig = al.align_fastx_text
        al.align_fastx_text = lambda *a, **kw: calls.append(len(a[0])) or orig(*a, **kw)
        seq = F.read_fasta(os.path.join(EX, GRAPHS[0][1]))[1][0] * 300
        big = str(tmp_path / "big.fa")
        open(big, "wb").write(b">long\n" + b"".join(seq[i:i + 60] + b"\n" for i in range(0, len(seq), 60))
                              + b">short\n" + seq[:40] + b"\n")
        whole, small = io.BytesIO(), io.BytesIO()
        cli.align_file(al, big, whole)
        del calls[:]
        cli.align_file(al, big, small, chunk_bytes=97)
        assert small.getvalue() == whole.getvalue() and whole.getvalue().count(b"\n") == 2
        assert len(calls) <= 14, calls                     # 11 kB in 97-byte chunks: 8 doublings, not 114 parses
        bad = str(tmp_path / "bad.fq")
        good = b"@r1\n" + seq[:50] + b"\n+\n" + b"I" * 50 + b"\n"
        open(bad, "wb").write(good + b"@r2\nACGT\n+\nII\n" + good * 20000)
        out = io.BytesIO()
        del calls[:]
        cli.align_file(al, bad, out, chunk_bytes=4096)
        assert len(calls) == 1                             # no chunk after the one that ended the file
        exp = io.BytesIO()
        one = str(tmp_path / "one.fq")
        open(one, "wb").write(good)
        cli.align_file(al, one, exp)
        assert out.getvalue() == exp.getvalue()
    finally:
        idx.close()
