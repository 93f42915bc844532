"""`metagraph_b200 align --distributed` and sharding.align_sharded_text on the device, with two gloo ranks on device 0
(gloo carries the token and the text): C2- and C3-shaped FASTQ of 100 k reads, plain, BGZF and plain gzip, give the
bytes `--devices 0` gives, TSV and JSON; align_sharded_text equals align_batch_text on one rank."""
import os
import socket
import subprocess
import sys

import pytest

import bench
import bgzf_common as B
import fastx_common as F
from test_gzip_gpu import gz

pytestmark = pytest.mark.gpu

N = 100_000

# every rank builds the graph of bench's 2 Mbp genome in place of loading a .dbg, and runs the command or the API
WORKER = r'''
import os, sys
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import bench
from metagraph_b200 import cli
from metagraph_b200.aligner import B200Aligner, BOSSTable, DBGSuccinctIndex
genome = bench.make_genome(2_000_000)
boss = BOSSTable.from_sequences(31, [genome.tobytes().decode()])
BOSSTable.from_dbg = classmethod(lambda cls, path, lib=None: boss)
if sys.argv[1] == "align":
    cli.CHUNK_BYTES = int(os.environ["MGB_TEST_CHUNK"])
    sys.exit(cli.main(sys.argv[1:]))
import torch.distributed as dist
from test_multi_device_gpu import shaped_reads
from metagraph_b200.sharding import align_sharded_text
dist.init_process_group("gloo")
idx = DBGSuccinctIndex(boss, device=0)
n, L = 20000, bench.READ_LEN
for shape, (buf, cfg) in shaped_reads(genome, n).items():
    al = B200Aligner(idx, cfg)
    batch = [(b"r%d" % i, buf[i * L:(i + 1) * L].tobytes()) for i in range(n)]
    for json in (False, True):
        got = align_sharded_text(al, batch, json)
        if dist.get_rank() == 0:
            exp = al.align_batch_text(batch, json)
            assert got == exp and exp.count(b"\n") >= n, (shape, json)
        else:
            assert got is None
idx.close()
print("SHARDED_TEXT_OK")
dist.destroy_process_group()
'''


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _env(chunk=0):
    env = dict(os.environ, MGB_TEST_CHUNK=str(chunk), MASTER_ADDR="127.0.0.1", OMP_NUM_THREADS="1")
    env.pop("MGB_LIB", None)
    # both ranks on the first visible device
    env["CUDA_VISIBLE_DEVICES"] = os.environ.get("CUDA_VISIBLE_DEVICES", "0").split(",")[0]
    return env


def _torchrun(worker, argv, env):
    return subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
                           "--master-addr", "127.0.0.1", "--master-port", str(_free_port()), worker] + argv,
                          capture_output=True, env=env, timeout=1800)


@pytest.fixture(scope="module")
def worker(tmp_path_factory):
    p = tmp_path_factory.mktemp("worker") / "worker.py"
    p.write_text("ROOT = %r\n" % F.ROOT + WORKER)
    return str(p)


@pytest.mark.parametrize("shape", ["c2", "c3"])
def test_two_ranks_match_one_device(worker, shape, tmp_path):
    from test_multi_device_gpu import shaped_reads
    genome = bench.make_genome(2_000_000)
    buf, _ = shaped_reads(genome, N)[shape]
    data = B.fastq_of(buf.reshape(N, bench.READ_LEN))
    paths = [str(tmp_path / "r.fq"), str(tmp_path / "r.fq.bgz"), str(tmp_path / "r.fq.gz")]
    for p, b in zip(paths, (data, B.write(data), gz(data, 6))):
        open(p, "wb").write(b)
    env = _env(len(data) // 12)
    argv = ["-i", "graph.dbg"] + (["--align-min-seed-length", "31", "--align-max-seed-length", "31"]
                                  if shape == "c2" else ["--align-min-exact-match", "0"])
    for fmt in ([], ["--json"]):
        one = subprocess.run([sys.executable, worker, "align", "--devices", "0"] + argv + fmt + paths,
                             capture_output=True, env=env, timeout=1800)
        assert one.returncode == 0, one.stderr[-3000:]
        assert one.stdout.count(b"\n") >= 3 * N
        two = _torchrun(worker, ["align", "--distributed"] + argv + fmt + paths, env)
        assert two.returncode == 0, two.stderr[-3000:]
        assert two.stdout == one.stdout, (shape, fmt)


def test_align_sharded_text(worker):
    r = _torchrun(worker, ["sharded"], _env())
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-3000:]
    assert b"SHARDED_TEXT_OK" in r.stdout
