"""SAM and BAM files split among shards (jellyfish_b200/split_sam.py) on one H100: one engine per shard, as the multi-GPU
path runs them.  Each shard stages its share piece by piece into FASTQ (jfgpu_sam_stage) and routes it as FASTQ through the
key exchange (jfgpu_extract_route) or the record exchange (jfgpu_shard_*).  The concatenated shard dumps must be the FASTQ
golden databases byte for byte, whatever the form of the file (SAM, gzip'd SAM, BAM).  A BAM whose cut is fooled by an
imitated record chain must be caught and counted whole, exactly; a malformed record is an error with its byte offset.
`count_multi --sam` runs as a command in one process, and under torchrun when there are at least 2 GPUs."""
import gzip
import json
import os
import subprocess
import sys

import pytest

import jfutil
import sam_tools
from cases import CASES

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = json.load(open(os.path.join(HERE, "golden", "golden.json")))
PIECE = 40000             # small pieces: every share is staged in several calls, records straddle them
FORMS = ("sam", "sam.gz", "bam")


def _size(v):
    return int(v[:-1]) * {"k": 10**3, "M": 10**6, "G": 10**9}[v[-1]] if v[-1] in "kMG" else int(v)


def _forms(workdir, inputs, name, block=7000):
    base = os.path.join(workdir, "splitsam_%d_%s" % (block, name))
    if not os.path.exists(base + ".bam"):
        sam = sam_tools.fastq_to_sam(open(inputs[name], "rb").read())
        open(base + ".sam", "wb").write(sam)
        open(base + ".sam.gz", "wb").write(gzip.compress(sam))
        open(base + ".bam", "wb").write(sam_tools.bgzf(sam_tools.sam_to_bam(sam), block=block))
    return {f: base + "." + f for f in FORMS}


def _readers(path, rank, world):
    """The reader of `rank` and whether a failure of it falls back (split shares) or is an error (whole files)."""
    from jellyfish_b200 import split_sam
    k = split_sam.kind(path)
    if k in ("sam", "bam"):
        kind, share = split_sam.plan_file(path, rank, world, k)
        if kind == "sam":
            return split_sam.SamShareReader(path, share, PIECE), True
        return split_sam.BamShareReader(path, share, PIECE, threads=4), True
    return split_sam.WholeSamReader(path, rank == 0, PIECE), False


class _Shards(object):
    """`world` shard engines on one device and the key exchange between them, done by hand."""

    def __init__(self, k, size, canonical, world, bc=None, bf_size=0):
        import torch
        from jellyfish_b200 import HashCounter
        self.world = world
        self.hc = [HashCounter(size, 7, k=k, canonical=canonical, shard_index=r, n_shards=world, allow_regrow=False,
                               max_batch_bytes=1 << 20, bf_size=bf_size, bf_fp=0.01 if bf_size else 0.0) for r in range(world)]
        if bc:
            for hc in self.hc:
                hc.load_bloom_counter(bc)
        kw = self.hc[0].key_words
        self.cap = 2 * PIECE + (1 << 20) + 65536
        self.keys = torch.zeros((world, self.cap * kw), dtype=torch.int64, device="cuda")
        self.counts = torch.zeros(world, dtype=torch.int64, device="cuda")
        self.out_cap = 2 * (PIECE + (1 << 19)) + 64
        self.out = torch.zeros(self.out_cap, dtype=torch.uint8, device="cuda")

    def route(self, r, ptr, n):
        import torch
        self.counts.zero_()
        torch.cuda.synchronize()
        self.hc[r].extract_route(ptr, n, self.keys.data_ptr(), self.cap, self.counts.data_ptr(), begin=True, end=True, fmt="fastq")
        c = self.counts.tolist()
        for d in range(self.world):
            self.hc[d].insert_keys(self.keys[d].data_ptr(), c[d])
        torch.cuda.synchronize()

    def add(self, r, reader, tolerant):
        """-> False when a tolerant reader failed (its share must not count on its own)"""
        from jellyfish_b200 import JellyfishError, _lib
        try:
            for i in range(reader.n_pieces):
                data, begin, end = reader.read(i)
                reader.prefetch(i + 1)
                try:
                    n = self.hc[r].sam_stage(data, self.out.data_ptr(), self.out_cap, begin=begin, end=end, bam=reader.bam)
                except JellyfishError as ex:
                    if tolerant and ex.code == _lib.ERR_FORMAT:
                        return False
                    raise
                reader.release(i)
                if n:
                    self.route(r, self.out.data_ptr(), n)
            return True
        finally:
            reader.close()

    def count(self, paths):
        """split every file; on a failed share clear and count whole files (rank i % world) -> (header, body, fell back)"""
        from jellyfish_b200 import split_sam
        ok = all([self.add(r, *_readers(p, r, self.world)) for p in paths for r in range(self.world)])
        if not ok:
            for hc in self.hc:
                hc.clear()
            for i, p in enumerate(paths):
                self.add(i % self.world, split_sam.WholeSamReader(p, True, PIECE), False)
        return self.dump() + (not ok,)

    def dump(self):
        from jellyfish_b200.distributed import concat_shards
        import tempfile
        with tempfile.TemporaryDirectory() as d:
            out = os.path.join(d, "split")
            for r, hc in enumerate(self.hc):
                hc.done()
                hc.dump("%s.%d" % (out, r))
                hc.close()
            return jfutil.split_db(concat_shards(out, self.world, out + ".jf"))


@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("world", [2, 4, 8])
@pytest.mark.parametrize("name", ["fq", "fq_k63", "fq_long"])
def test_split_sam_key_exchange(name, world, form, built, workdir, inputs):
    args, ins = CASES[name]
    g = GOLDEN[name]
    paths = [_forms(workdir, inputs, i)[form] for i in ins]
    sh = _Shards(int(args[args.index("-m") + 1]), _size(args[args.index("-s") + 1]), "-C" in args, world)
    h, b, fell = sh.count(paths)
    assert not fell
    assert jfutil.semantic(h) == g["header"]
    assert jfutil.md5(b) == g["body_md5"]


def _one_gpu_count(workdir, tag, args, sams=(), files=()):
    db = os.path.join(workdir, "splitsam_ref_%s.jf" % tag)
    cmd = [jfutil.OUR_JF, "count"] + list(args) + ["-o", db] + list(files)
    for s in sams:
        cmd += ["--sam", s]
    jfutil.run(cmd, timeout=900)
    return jfutil.split_db(db)


def test_split_sam_k100(built, workdir, inputs):
    """k = 100 (four-word keys): the split count of a BAM and of SAM text against the single-GPU `count --sam`."""
    args = ["-m", "100", "-s", "1M", "-C"]
    f = _forms(workdir, inputs, "reads.fq")
    h1, b1 = _one_gpu_count(workdir, "k100", args, sams=[f["bam"]])
    for form in ("bam", "sam"):
        sh = _Shards(100, _size("1M"), True, 4)
        h, b, fell = sh.count([f[form]])
        assert not fell and b == b1 and b


def test_split_sam_record_exchange(built, workdir, inputs):
    """k = 17 through the record exchange: the FASTQ of every piece goes through jfgpu_shard_extract as a file of its own."""
    import torch
    from jellyfish_b200 import HashCounter
    from jellyfish_b200.distributed import CHUNK
    world = 2
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    arena = 2 * n_sm * max(1, 1024 // world) + 64
    shards, bufs = [], []
    for r in range(world):
        hc = HashCounter(_size("600k"), 7, k=17, canonical=True, shard_index=r, n_shards=world, allow_regrow=False, part_min_mb=1,
                         pool_bytes=2 << 30, max_batch_bytes=1 << 20)
        bb = [torch.empty(2 * world * arena * CHUNK, dtype=torch.uint8, device="cuda"), torch.empty(2 * world * arena * 8, dtype=torch.uint8, device="cuda"),
              torch.empty(world * arena * CHUNK, dtype=torch.uint8, device="cuda"), torch.empty(world * arena * 8, dtype=torch.uint8, device="cuda")]
        assert hc.shard_setup(bb[0].data_ptr(), bb[1].data_ptr(), arena, bb[2].data_ptr(), bb[3].data_ptr(), arena)
        shards.append(hc)
        bufs.append(bb)
    out_cap = 2 * (PIECE + (1 << 19)) + 64
    out = torch.zeros(out_cap, dtype=torch.uint8, device="cuda")
    f = _forms(workdir, inputs, "reads.fq")
    n_round = [0]
    for form in ("bam", "sam"):
        for r in range(world):
            reader, _ = _readers(f[form], r, world)
            for i in range(reader.n_pieces):
                data, begin, end = reader.read(i)
                n = shards[r].sam_stage(data, out.data_ptr(), out_cap, begin=begin, end=end, bam=reader.bam)
                if not n:
                    continue
                bank = n_round[0] & 1
                n_round[0] += 1
                shards[r].shard_extract(out.data_ptr(), n, bank, begin=True, end=True, fmt="fastq")
                counts = shards[r].shard_pack(bank)
                for d in range(world):
                    c = counts[d]
                    a0 = (bank * world + d) * arena
                    bufs[d][2][r * arena * CHUNK:(r * arena + c) * CHUNK] = bufs[r][0][a0 * CHUNK:(a0 + c) * CHUNK]
                    bufs[d][3][r * arena * 8:(r * arena + c) * 8] = bufs[r][1][a0 * 8:(a0 + c) * 8]
                    torch.cuda.synchronize()
                    got = [0] * world
                    got[r] = c
                    shards[d].shard_unpack(got)
                    torch.cuda.synchronize()
            reader.close()
    from jellyfish_b200.distributed import concat_shards
    out_path = os.path.join(workdir, "splitsam_rx")
    for r, hc in enumerate(shards):
        hc.done()
        hc.dump("%s.%d" % (out_path, r))
        hc.close()
    h, b = jfutil.split_db(concat_shards(out_path, world, out_path + ".jf"))
    # both forms were counted: every count is twice the golden one
    hg, bg = _one_gpu_count(workdir, "rx", ["-m", "17", "-s", "600k", "-C"], files=[inputs["reads.fq"], inputs["reads.fq"]])
    assert b == bg


def test_fooled_bam_cut_falls_back_exactly(built, workdir):
    """The imitated record chain of test_split_sam_cpu: rank 1 starts on it, rank 0's records then end past rank 1's
    start, the share is refused and every file is counted whole -- the same database as one GPU."""
    import test_split_sam_cpu as cpu
    data, fake_at, stream = cpu.imitation_bam()
    path = os.path.join(workdir, "splitsam_fooled.bam")
    open(path, "wb").write(data)
    args = ["-m", "21", "-s", "1M", "-C"]
    hr, br = _one_gpu_count(workdir, "fooled", args, sams=[path])
    sh = _Shards(21, _size("1M"), True, 2)
    h, b, fell = sh.count([path])
    assert fell and b == br and b


def test_malformed_record_is_an_error_with_its_offset(built, workdir, inputs):
    from jellyfish_b200 import JellyfishError
    sam = sam_tools.fastq_to_sam(open(inputs["reads.fq"], "rb").read())
    lines = sam.split(b"\n")
    bad = 2000
    at = len(b"\n".join(lines[:bad])) + 1
    lines[bad] = b"\t".join(lines[bad].split(b"\t")[:9])
    path = os.path.join(workdir, "splitsam_bad.sam")
    open(path, "wb").write(b"\n".join(lines))
    sh = _Shards(21, _size("1M"), True, 4)
    with pytest.raises(JellyfishError) as ex:
        sh.count([path])
    assert "Invalid SAM line at byte %d of the file: fewer than 11 fields" % at in str(ex.value)
    # the command writes no output
    out = os.path.join(workdir, "splitsam_bad.jf")
    r = _run_multi(1, ["-m", "21", "-s", "1M", "-C", "-o", out, "--sam", path], check=False)
    assert r.returncode != 0 and "byte %d" % at in r.stdout.decode(errors="replace") and not os.path.exists(out)


def test_split_sam_bloom_counter(built, workdir, inputs):
    """--bc through the key exchange, byte for byte with the single-GPU `count --bc --sam`."""
    bcf = os.path.join(workdir, "splitsam.bc")
    jfutil.run([jfutil.OUR_JF, "bc", "-m", "21", "-s", "1M", "-C", "-o", bcf, inputs["reads.fq"]], timeout=600)
    f = _forms(workdir, inputs, "reads.fq")
    args = ["-m", "21", "-s", "1M", "-C", "--bc", bcf]
    hr, br = _one_gpu_count(workdir, "bc", args, sams=[f["bam"]])
    for world in (2, 4):
        sh = _Shards(21, _size("1M"), True, world, bc=bcf)
        h, b, fell = sh.count([f["bam"]])
        assert not fell and b == br


def test_split_sam_bloom_prefilter(built, workdir, inputs):
    """--bf-size: the filter drops at most the first occurrence of a k-mer, and keeps every k-mer seen twice or more."""
    f = _forms(workdir, inputs, "reads.fq")
    hr, br = _one_gpu_count(workdir, "occ", ["-m", "21", "-s", "1M", "-C"], files=[inputs["reads.fq"]])
    occ = dict(jfutil.records(hr, br))
    sh = _Shards(21, _size("1M"), True, 4, bf_size=1000000)
    h, b, fell = sh.count([f["bam"]])
    got = dict(jfutil.records(h, b))
    assert not fell and set(got) <= set(occ)
    assert all(v in (occ[k], occ[k] - 1) for k, v in got.items())
    assert all(k in got for k, v in occ.items() if v > 1)


def _run_multi(world, args, port=29771, check=True):
    env = dict(os.environ, SOURCE_DATE_EPOCH="0")
    for v in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        env.pop(v, None)
    if world == 1:
        cmd = [sys.executable, "-m", "jellyfish_b200.count_multi"] + args
    else:
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(world), "--master-addr",
               "127.0.0.1", "--master-port", str(port), "-m", "jellyfish_b200.count_multi"] + args
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, timeout=600, cwd=jfutil.ROOT, env=env)
    if check:
        assert r.returncode == 0, r.stdout.decode(errors="replace")[-3000:]
    return r


def test_count_multi_sam_one_process(built, workdir, inputs):
    """count_multi --sam in one process, with positional FASTA first, --split auto and files, against `count --sam`."""
    f = _forms(workdir, inputs, "reads.fq")
    g = _forms(workdir, inputs, "reads_q.fq")
    args = ["-m", "31", "-s", "2M", "-C"]
    sams = [f["bam"], g["sam"], f["sam.gz"]]
    hr, br = _one_gpu_count(workdir, "cm1", args, sams=sams, files=[inputs["multi.fa"]])
    for split in ("auto", "files"):
        out = os.path.join(workdir, "splitsam_cm1_%s.jf" % split)
        cmd = args + ["--split", split, "-o", out, inputs["multi.fa"]]
        for s in sams:
            cmd += ["--sam", s]
        _run_multi(1, cmd)
        assert jfutil.split_db(out)[1] == br, split


def _ngpu():
    try:
        import torch
        return torch.cuda.device_count()
    except Exception:
        return 0


def test_count_multi_sam_two_ranks_on_one_gpu(built, workdir, inputs):
    """The production path of several ranks (split plan, streamed pieces, ShardedCounter.add_sam_pieces with the key
    exchange, the check after the count and its fall-back, `--split files` through the block-by-block whole-file reader)
    with two ranks on one device, joined by gloo (tests/sam_ranks_worker.py): the output of `count --sam`, byte for byte."""
    import test_split_sam_cpu as cpu
    f = _forms(workdir, inputs, "reads.fq")
    g = _forms(workdir, inputs, "reads_q.fq")
    fooled = os.path.join(workdir, "splitsam_fooled_2r.bam")
    open(fooled, "wb").write(cpu.imitation_bam()[0])
    worker = os.path.join(HERE, "sam_ranks_worker.py")
    env = dict(os.environ, SOURCE_DATE_EPOCH="0")
    for v in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        env.pop(v, None)
    for i, (k, sams, split) in enumerate(((21, [f["bam"], g["sam"], f["sam.gz"]], "auto"), (21, [f["bam"], g["bam"]], "files"),
                                          (100, [f["bam"]], "auto"), (21, [fooled, g["sam"]], "auto"))):
        args = ["-m", str(k), "-s", "1M", "-C"]
        hr, br = _one_gpu_count(workdir, "2r%d" % i, args, sams=sams)
        out = os.path.join(workdir, "splitsam_2r_%d.jf" % i)
        cmd = args + ["--split", split, "-o", out]
        for s_ in sams:
            cmd += ["--sam", s_]
        r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr",
                            "127.0.0.1", "--master-port", str(29790 + i), worker] + cmd,
                           stdout=subprocess.PIPE, stderr=subprocess.STDOUT, timeout=600, cwd=jfutil.ROOT, env=env)
        log = r.stdout.decode(errors="replace")
        assert r.returncode == 0, log[-3000:]
        assert "rank 1 --sam times" in log and "2 GPUs" in log, log[-3000:]
        assert jfutil.split_db(out)[1] == br and br, (k, sams, split)
        assert ("counting whole files per rank instead" in log) == (sams[0] == fooled), log[-3000:]


@pytest.mark.skipif(_ngpu() < 2, reason="needs at least 2 GPUs")
def test_count_multi_sam_under_torchrun(built, workdir, inputs):
    import test_split_sam_cpu as cpu
    world = 2
    f = _forms(workdir, inputs, "reads.fq")
    fooled = os.path.join(workdir, "splitsam_fooled_tr.bam")
    open(fooled, "wb").write(cpu.imitation_bam()[0])
    for k, sams in ((21, [f["bam"], f["sam"], f["sam.gz"]]), (100, [f["bam"]]), (17, [f["sam"]]), (21, [fooled])):
        args = ["-m", str(k), "-s", "4M" if k == 17 else "1M", "-C"]
        hr, br = _one_gpu_count(workdir, "tr%d" % k, args, sams=sams)
        out = os.path.join(workdir, "splitsam_tr_%d.jf" % k)
        cmd = args + ["-o", out]
        for s in sams:
            cmd += ["--sam", s]
        r = _run_multi(world, cmd)
        assert jfutil.split_db(out)[1] == br, (k, sams)
        if sams == [fooled]:
            assert b"counting whole files per rank instead" in r.stdout
