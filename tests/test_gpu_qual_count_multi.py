"""`count_multi` with -Q / --min-quality and --if end to end, against the single-GPU `count` of the command-line driver and
the reference's goldens.  World 1 runs on any H100 (the split path streams every file through record-aligned pieces);
the torchrun cases need at least 2 GPUs.  Errors are only provoked at world 1, where no peer can be left waiting."""
import json
import os
import subprocess
import sys

import pytest

import jfutil
from cases import CASES, QUAL_CASES
from test_gpu_split_multi import _fooled_fastq, _multi, _ngpu, _one_gpu

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(__file__)
GOLDEN = json.load(open(os.path.join(HERE, "golden", "golden.json")))
GOLDEN_QUAL = json.load(open(os.path.join(HERE, "golden", "golden_qual.json")))
NAMES = sorted(n for n in QUAL_CASES if n not in ("q_ml", "q_mixed")) + ["if_sub", "if_zeros", "if_k40_rep"]


def _args(name, inputs):
    args, ins = CASES[name] if name in CASES else QUAL_CASES[name]
    return jfutil.subst(list(args), inputs), [inputs[f] for f in ins]


@pytest.mark.parametrize("name", NAMES)
def test_world_1_matches_count(name, built, workdir, inputs):
    args, files = _args(name, inputs)
    ref = os.path.join(workdir, "qm_ref_%s.jf" % name)
    ref_b = _one_gpu("count", args, ref, files)
    ref_h = jfutil.split_db(ref)[0]
    for split in ("auto", "files"):
        out = os.path.join(workdir, "qm_%s_%s.jf" % (name, split))
        b, _ = _multi(1, "count_multi", args, out, files, split, 0)
        assert b == ref_b, split
        assert jfutil.semantic(jfutil.split_db(out)[0]) == jfutil.semantic(ref_h)


def test_sam_with_quality_matches_count(built, workdir, inputs):
    """--sam with -Q: the FASTQ the transcode writes is whole records, counted as the single-GPU `count --sam -Q` counts."""
    fq = inputs["reads_q.fq"]
    sam = os.path.join(workdir, "qm_reads_q.sam")
    with open(sam, "wb") as f:
        f.write(_to_sam(open(fq, "rb").read()))
    for args in (["-m", "21", "-s", "1M", "-C", "-Q", "5"], ["-m", "17", "-s", "1M", "--min-quality", "20", "--quality-start", "33"]):
        ref = _one_gpu("count", args + ["--sam", sam], os.path.join(workdir, "qm_sam_ref.jf"), [inputs["multi.fa"]])
        for split in ("auto", "files"):
            b, _ = _multi(1, "count_multi", args + ["--sam", sam], os.path.join(workdir, "qm_sam_%s.jf" % split), [inputs["multi.fa"]], split, 0)
            assert b == ref, (args, split)


def _to_sam(fq):
    lines = fq.split(b"\n")
    out = [b"@HD\tVN:1.6"]
    for i in range(0, len(lines) - 3, 4):
        out.append(b"\t".join([lines[i][1:] or b"r", b"4", b"*", b"0", b"0", b"*", b"*", b"0", b"0", lines[i + 1] or b"*",
                               lines[i + 3] or b"*"]))
    return b"\n".join(out) + b"\n"


@pytest.mark.parametrize("name", ["q_ml", "q_mixed"])
def test_multi_line_fastq_fails_as_on_one_gpu(name, built, workdir, inputs):
    args, files = _args(name, inputs)
    for split in ("auto", "files"):
        env = dict(os.environ, SOURCE_DATE_EPOCH="0")
        for v in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
            env.pop(v, None)
        r = subprocess.run([sys.executable, "-m", "jellyfish_b200.count_multi"] + args + ["--split", split, "-o",
                           os.path.join(workdir, "qm_ml.jf")] + files, stdout=subprocess.PIPE, stderr=subprocess.PIPE,
                           cwd=jfutil.ROOT, env=env, timeout=600)
        assert r.returncode != 0 and b"Invalid fastq" in r.stderr, (split, r.stderr[-2000:])


def test_bad_quality_switches_exit_before_counting(built, workdir, inputs):
    for sw, msg in ((["-Q", "ab"], b"Error: [-Q, --min-qual-char] must be one character."),
                    (["--min-quality", "63"], b"Error: Min quality 63 is outside the range [0, 62]")):
        r = subprocess.run([sys.executable, "-m", "jellyfish_b200.count_multi", "-m", "21", "-s", "1M"] + sw +
                           ["-o", os.path.join(workdir, "qm_bad.jf"), inputs["reads_q.fq"]], stderr=subprocess.PIPE,
                           cwd=jfutil.ROOT, timeout=600)
        assert r.returncode == 1 and msg in r.stderr


def test_two_ranks_on_one_gpu(built, workdir, inputs):
    """The production path of several ranks with two ranks on one device, joined by gloo (tests/qual_ranks_worker.py), and
    rounds of 200 KB: the split plan, ShareReader(records=True), ShardedCounter.add_device_text(fastq=True) with its
    record-aligned rounds copied to aligned staging, the two passes of --if and the fall-back that repeats both.  The
    output of the single-GPU `count`, byte for byte."""
    from test_gpu_split_multi import _fooled_fastq
    fq = os.path.join(workdir, "qm2r_fooled.fq")
    with open(fq, "wb") as fh:
        fh.write(_fooled_fastq(2, 21))
    fooled = (["-m", "21", "-s", "1M", "-C", "-Q", "5", "--if", fq], [fq, inputs["reads_q.fq"]])
    runs = [(_args("q_fq", inputs), "auto"), (_args("q_fq", inputs), "files"), (_args("q_dos", inputs), "files"),
            (_args("q_fa", inputs), "auto"), (_args("if_sub", inputs), "auto"), (_args("if_sub", inputs), "files"),
            (_args("q_k40_if", inputs), "auto"), (fooled, "auto")]
    worker = os.path.join(HERE, "qual_ranks_worker.py")
    env = dict(os.environ, SOURCE_DATE_EPOCH="0")
    for v in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        env.pop(v, None)
    for i, ((args, files), split) in enumerate(runs):
        ref = _one_gpu("count", args, os.path.join(workdir, "qm2r_ref_%d.jf" % i), files)
        out = os.path.join(workdir, "qm2r_%d.jf" % i)
        r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr",
                            "127.0.0.1", "--master-port", str(29870 + i), worker, "200000"] + args + ["--split", split, "-o", out] + files,
                           stdout=subprocess.PIPE, stderr=subprocess.STDOUT, timeout=600, cwd=jfutil.ROOT, env=env)
        log = r.stdout.decode(errors="replace")
        assert r.returncode == 0, log[-3000:]
        assert "2 GPUs" in log, log[-3000:]
        assert jfutil.split_db(out)[1] == ref and ref, (args, split)
        assert ("counting whole files per rank instead" in log) == (args is fooled[0]), log[-3000:]


@pytest.mark.skipif(_ngpu() < 2, reason="needs at least 2 GPUs")
@pytest.mark.parametrize("world", [2, 4, 8])
def test_quality_and_if_under_torchrun(world, built, workdir, inputs):
    if _ngpu() < world:
        pytest.skip("needs %d GPUs" % world)
    port = 29780 + 10 * world
    for j, name in enumerate(("q_fq", "q_k40_if", "if_sub")):
        args, files = _args(name, inputs)
        g = GOLDEN[name] if name in CASES else GOLDEN_QUAL[name]
        for split in ("auto", "files"):
            out = os.path.join(workdir, "qmw_%d_%s_%s.jf" % (world, name, split))
            b, _ = _multi(world, "count_multi", args, out, files, split, port + j)
            assert jfutil.md5(b) == g["body_md5"], (name, split)
            assert jfutil.semantic(jfutil.split_db(out)[0]) == g["header"]
    # a FASTQ file whose cut fools the local rule: both passes of --if are repeated with whole files
    fq = os.path.join(workdir, "qm_fooled_%d.fq" % world)
    with open(fq, "wb") as fh:
        fh.write(_fooled_fastq(world, 21))
    args = ["-m", "21", "-s", "1M", "-C", "-Q", "5", "--if", fq]
    ref = _one_gpu("count", args, os.path.join(workdir, "qmw_ref_fq.jf"), [fq, inputs["reads_q.fq"]])
    b, log = _multi(world, "count_multi", args, os.path.join(workdir, "qmw_%d_fq.jf" % world), [fq, inputs["reads_q.fq"]], "auto", port + 5)
    assert b == ref and "counting whole files per rank instead" in log
