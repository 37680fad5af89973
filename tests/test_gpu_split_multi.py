"""`count_multi` and `bc_multi` end to end on one input file, with `--split auto` and `--split files`, against the single-GPU
`count` / `bc` of the command-line driver.  One process (world 1) runs on any H100, a pipe included (process substitution:
the file is not split but read whole).  Under torchrun (worlds 2, 4, 8, skipped below that many GPUs) the key exchange,
the record exchange, `--bc` and a FASTQ file whose cut fools the local rule (the count falls back to whole files) are
covered."""
import os
import random
import subprocess
import sys

import pytest

import jfutil

pytestmark = pytest.mark.gpu


def _ngpu():
    try:
        import torch
        return torch.cuda.device_count()
    except Exception:
        return 0


def _run(cmd, world=1, port=29671, shell=False):
    env = dict(os.environ, SOURCE_DATE_EPOCH="0")
    for v in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        env.pop(v, None)
    if shell:
        r = subprocess.run(["bash", "-c", cmd], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, timeout=600, cwd=jfutil.ROOT, env=env)
    elif world == 1:
        r = subprocess.run([sys.executable, "-m"] + cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, timeout=600, cwd=jfutil.ROOT, env=env)
    else:
        r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(world),
                            "--master-addr", "127.0.0.1", "--master-port", str(port), "-m"] + cmd,
                           stdout=subprocess.PIPE, stderr=subprocess.STDOUT, timeout=600, cwd=jfutil.ROOT, env=env)
    assert r.returncode == 0, r.stdout.decode(errors="replace")[-3000:]
    return r.stdout.decode(errors="replace")


def _one_gpu(sub, args, out, files):
    jfutil.run([jfutil.OUR_JF, sub] + args + ["-o", out] + files, timeout=600)
    return jfutil.split_db(out)[1]


def _multi(world, module, args, out, files, split, port):
    log = _run(["jellyfish_b200." + module] + args + ["--split", split, "-o", out] + files, world, port)
    return jfutil.split_db(out)[1], log


def _fooled_fastq(world, k):
    """A FASTQ file (sequence lines that start with '@', quality lines that start with '+', headers as long as the '+'
    lines) whose first header is lengthened until some rank's cut lands in a header and takes the sequence line behind it."""
    from jellyfish_b200 import split
    rng = random.Random(3)
    recs = [b"@r\n@" + bytes(rng.choice(b"ACGT") for _ in range(60)) + b"\n+r\n+" + b"I" * 60 + b"\n" for _ in range(3000)]
    body = b"".join(recs[1:])
    for h in range(1, 400):
        data = b"@" + b"x" * h + recs[0][2:] + body
        rd = lambda off, n: data[off:off + n]
        shares = [split.plan_share(rd, len(data), "fastq", r, world, k) for r in range(world)]
        if not split.fastq_cuts_ok([(s.end - s.start, data[s.start:s.end].count(b"\n")) for s in shares]):
            return data
    raise AssertionError("no fooled cut found")


def test_count_multi_one_process(built, workdir, inputs):
    """World 1: the split path streams every file through the pinned pieces; the same database as `count`, also for a
    pipe (`<(cat FILE)`), which is read whole."""
    files = [inputs["multi.fa"], inputs["reads.fq"], inputs["dos.fa"]]
    args = ["-m", "31", "-s", "1M", "-C"]
    ref = _one_gpu("count", args, os.path.join(workdir, "sm1_ref.jf"), files)
    for split in ("auto", "files"):
        b, _ = _multi(1, "count_multi", args, os.path.join(workdir, "sm1_%s.jf" % split), files, split, 0)
        assert b == ref, split
    out = os.path.join(workdir, "sm1_pipe.jf")
    _run("python -m jellyfish_b200.count_multi %s -o %s %s <(cat %s) %s" % (" ".join(args), out, files[0], files[1], files[2]), shell=True)
    assert jfutil.split_db(out)[1] == ref


def test_bc_multi_one_process(built, workdir, inputs):
    files = [inputs["plain.fa"], inputs["reads.fq"]]
    args = ["-m", "21", "-s", "1M", "-C"]
    ref = _one_gpu("bc", args, os.path.join(workdir, "sm1_ref.bc"), files)
    for split in ("auto", "files"):
        b, _ = _multi(1, "bc_multi", args, os.path.join(workdir, "sm1_%s.bc" % split), files, split, 0)
        assert b == ref, split


@pytest.mark.skipif(_ngpu() < 2, reason="needs at least 2 GPUs")
@pytest.mark.parametrize("world", [2, 4, 8])
def test_one_file_under_torchrun(world, built, workdir, inputs):
    if _ngpu() < world:
        pytest.skip("needs %d GPUs" % world)
    port = 29680 + 10 * world
    # key exchange (k = 31 and k = 100) and record exchange (k = 17 with 4M slots: every shard filled region by region)
    for args, f in ((["-m", "31", "-s", "1M", "-C"], "plain1m.fa"), (["-m", "100", "-s", "1M", "-C"], "multi.fa"),
                    (["-m", "17", "-s", "4M", "-C"], "plain1m.fa"), (["-m", "21", "-s", "1M", "-C"], "reads.fq")):
        ref = _one_gpu("count", args, os.path.join(workdir, "smw_ref.jf"), [inputs[f]])
        for split in ("auto", "files"):
            b, _ = _multi(world, "count_multi", args, os.path.join(workdir, "smw_%d_%s.jf" % (world, split)), [inputs[f]], split, port)
            assert b == ref, (args, f, split)
    # bc across ranks, then count --bc through it
    bargs = ["-m", "21", "-s", "1M", "-C"]
    bc_ref = _one_gpu("bc", bargs, os.path.join(workdir, "smw_ref.bc"), [inputs["plain.fa"]])
    for split in ("auto", "files"):
        bcf = os.path.join(workdir, "smw_%d_%s.bc" % (world, split))
        b, _ = _multi(world, "bc_multi", bargs, bcf, [inputs["plain.fa"]], split, port + 1)
        assert b == bc_ref, split
    cargs = ["-m", "21", "-s", "1M", "-C", "--bc", bcf]
    ref = _one_gpu("count", cargs, os.path.join(workdir, "smw_ref_bc.jf"), [inputs["plain.fa"]])
    b, _ = _multi(world, "count_multi", cargs, os.path.join(workdir, "smw_%d_bc.jf" % world), [inputs["plain.fa"]], "auto", port + 2)
    assert b == ref
    # a FASTQ file that fools the local rule: the newline check fails and the files are counted whole
    fq = os.path.join(workdir, "fooled_%d.fq" % world)
    with open(fq, "wb") as fh:
        fh.write(_fooled_fastq(world, 21))
    args = ["-m", "21", "-s", "1M", "-C"]
    ref = _one_gpu("count", args, os.path.join(workdir, "smw_ref_fq.jf"), [fq])
    b, log = _multi(world, "count_multi", args, os.path.join(workdir, "smw_%d_fq.jf" % world), [fq], "auto", port + 3)
    assert b == ref and "counting whole files per rank instead" in log
    bc_ref = _one_gpu("bc", args, os.path.join(workdir, "smw_ref_fq.bc"), [fq])
    b, log = _multi(world, "bc_multi", args, os.path.join(workdir, "smw_%d_fq.bc" % world), [fq], "auto", port + 4)
    assert b == bc_ref and "counting whole files per rank instead" in log
