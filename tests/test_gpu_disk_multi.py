"""`count --disk` on shards: a full shard is written out (the spill hook, jfgpu_set_spill) and zeroed, counting goes on, and
each rank merges its own pieces; the rank-ordered concatenation is the single-GPU `count --disk` output, held to the
reference's goldens (golden_disk.json, golden_large_k.json).  World 1 and the emulated shards (every shard's engine on one
device, routed by extract_route / insert_keys as the key exchange routes them) run on one H100; the torchrun cases need
as many GPUs as ranks."""
import json
import os
import subprocess
import sys

import pytest

import gen
import jfutil
from cases import DISK_CASES, QUAL_CASES
from test_gpu_shard_large_k import _cuts
from test_gpu_split_multi import _fooled_fastq, _ngpu, _one_gpu, _run

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN_DISK = json.load(open(os.path.join(HERE, "golden", "golden_disk.json")))
GOLDEN_LK = json.load(open(os.path.join(HERE, "golden", "golden_large_k.json")))
UINT64_MAX = (1 << 64) - 1
# the disk goldens: (count switches, inputs, golden {header, body_md5[, body_len]})
CASES = {n: (DISK_CASES[n][0], DISK_CASES[n][1], GOLDEN_DISK[n]) for n in DISK_CASES}
CASES["k100C_disk"] = (GOLDEN_LK["cases"]["k100C_disk"]["args"], GOLDEN_LK["cases"]["k100C_disk"]["inputs"], GOLDEN_LK["cases"]["k100C_disk"])
SEQ1M = "seq1m"          # s2k_disk: -m 100 -s 2k --disk on 10000 lines of the reference's generated sequence
CASES["s2k_disk"] = (["-m", "100"] + GOLDEN_LK["large_key"]["s2k_disk"]["args"], [SEQ1M], GOLDEN_LK["large_key"]["s2k_disk"])


@pytest.fixture(scope="module")
def files(workdir, inputs):
    p = os.path.join(workdir, "disk_seq1m_0_10001.fa")
    if not os.path.exists(p):
        gen.generate_sequence_fasta(p + ".full", 1040104553, 1000000)
        with open(p + ".full", "rb") as f:
            lines = f.read().split(b"\n")
        with open(p, "wb") as f:
            f.write(b"\n".join(lines[:10001]) + b"\n")
    return dict(inputs, **{SEQ1M: p})


def _size(v):
    return int(v[:-1]) * {"k": 10**3, "M": 10**6, "G": 10**9}[v[-1]] if v[-1] in "kMG" else int(v)


def _opts(args):
    """-> (size, engine keyword arguments, (lower, upper), out_counter_len) of a case's count switches"""
    rest = [a for a in args if a not in ("-C", "--disk")]
    o = dict(zip(rest[0::2], rest[1::2]))
    eng = {"k": int(o["-m"]), "canonical": "-C" in args, "val_len": int(o.get("-c", 7))}
    if "-Q" in o:
        eng["min_qual"] = o["-Q"]
    if "--bf-size" in o:
        eng["bf_size"] = _size(o["--bf-size"])
    return _size(o["-s"]), eng, (int(o.get("-L", 0)), int(o.get("-U", UINT64_MAX))), int(o.get("--out-counter-len", 4))


def _check(h, b, g):
    assert jfutil.semantic(h) == g["header"]
    assert jfutil.md5(b) == g["body_md5"]
    if "body_len" in g:
        assert len(b) == g["body_len"]


@pytest.mark.parametrize("name", sorted(CASES))
def test_world_1_count_multi_disk_matches_golden(name, built, workdir, files):
    """count_multi --disk with one rank: at least two pieces, none left behind, the golden header and body; with --no-merge
    the pieces hold the golden records (summed and clipped as the merge does)."""
    args, ins, g = CASES[name]
    paths = [files[i] for i in ins]
    out = os.path.join(workdir, "dm1_%s.jf" % name)
    log = _run(["jellyfish_b200.count_multi"] + args + ["--disk", "-o", out] + paths)
    spills = int(log.split("--disk: spills ")[1].split()[0])
    assert spills >= 1, log                          # (at least two pieces: the spills and the table at the end)
    h, b = jfutil.split_db(out)
    _check(h, b, g)
    assert not [f for f in os.listdir(workdir) if f.startswith(os.path.basename(out) + ".")]
    out2 = os.path.join(workdir, "dm1nm_%s.jf" % name)
    _run(["jellyfish_b200.count_multi"] + args + ["--disk", "--no-merge", "-o", out2] + paths)
    assert not os.path.exists(out2)
    pieces = ["%s.0.%d" % (out2, i) for i in range(spills + 1)]
    assert all(os.path.exists(p) for p in pieces) and not os.path.exists("%s.0.%d" % (out2, spills + 1))
    total = {}
    for p in pieces:
        hp, bp = jfutil.split_db(p)
        assert hp["size"] == h["size"] and hp["matrix1"] == h["matrix1"]
        for key, v in jfutil.records(hp, bp):
            total[key] = total.get(key, 0) + v
        os.unlink(p)
    lo = int(args[args.index("-L") + 1]) if "-L" in args else 0
    cap = (1 << (8 * h["counter_len"])) - 1
    assert {key: min(v, cap) for key, v in total.items() if v >= lo} == dict(jfutil.records(h, b))


class DiskShards(object):
    """`world` engines of one global table on the current device, each with a spill hook (DiskPieces), fed through
    extract_route / insert_keys.  `fail_group` keys at most fail between two looks of the engine (max_batch_bytes)."""

    def __init__(self, size, world, out, ocl, cap, fail_group=4096, **eng):
        import torch
        from jellyfish_b200 import HashCounter
        from jellyfish_b200.distributed import DiskPieces
        val_len = eng.pop("val_len", 7)
        self.world, self.cap, self.fail_group = world, cap, fail_group
        self.hcs = [HashCounter(size, val_len, shard_index=r, n_shards=world, allow_regrow=False, max_batch_bytes=fail_group, **eng)
                    for r in range(world)]
        self.disk = [DiskPieces(hc, out, r, ocl) for r, hc in enumerate(self.hcs)]
        kw = self.hcs[0].key_words
        self.kw = kw
        self.keys = torch.zeros((world, cap * kw), dtype=torch.int64, device="cuda")
        self.counts = torch.zeros(world, dtype=torch.int64, device="cuda")
        self.local_slots = self.hcs[0].info()["local_slots"]
        self.most_failing = 0        # the most keys one insert_keys call handed a shard that cannot all have found a slot
        self.n_files = 0

    def add(self, data, chunk, fastq_records=False):
        import torch
        router = self.hcs[self.n_files % self.world]
        self.n_files += 1
        bounds = [0] + _cuts(data, chunk, fastq_records) + [len(data)]
        for a, b in zip(bounds[:-1], bounds[1:]):
            buf = torch.zeros(b - a + 256, dtype=torch.uint8, device="cuda")
            if b > a:
                buf[:b - a] = torch.frombuffer(bytearray(data[a:b]), dtype=torch.uint8).cuda()
            self.counts.zero_()
            torch.cuda.synchronize()
            router.extract_route(buf.data_ptr(), b - a, self.keys.data_ptr(), self.cap, self.counts.data_ptr(), begin=a == 0, end=b >= len(data))
            c = self.counts.tolist()
            assert max(c) <= self.cap
            for d in range(self.world):
                if c[d]:
                    distinct = torch.unique(self.keys[d, :c[d] * self.kw].view(-1, self.kw), dim=0).shape[0]
                    self.most_failing = max(self.most_failing, distinct - self.local_slots)
                self.hcs[d].insert_keys(self.keys[d].data_ptr(), c[d])

    def write(self, out, lower=0, upper=UINT64_MAX):
        from jellyfish_b200.distributed import concat_shards
        for r, hc in enumerate(self.hcs):
            hc.done()
            self.disk[r].write_output("%s.%d" % (out, r), lower, upper)
            assert not any(os.path.exists(p) for p in self.disk[r].pieces)
        return jfutil.split_db(concat_shards(out, self.world, out + ".jf"))

    def close(self):
        for hc in self.hcs:
            hc.close()


def _emulate(args, paths, world, out, chunk=400000):
    size, eng, (lo, hi), ocl = _opts(args)
    sh = DiskShards(size, world, out, ocl, cap=chunk + 65536, **eng)
    try:
        for p in paths:
            data = open(p, "rb").read()
            sh.add(data, chunk, fastq_records="min_qual" in eng and data[:1] == b"@")
        h, b = sh.write(out, lo, hi)
        spills = [len(d.pieces) - 1 for d in sh.disk]
        return h, b, spills, sh
    finally:
        sh.close()


@pytest.mark.parametrize("world", [2, 4, 8])
@pytest.mark.parametrize("name", ["disk_k17_c3", "disk_k21_LU", "disk_k40", "k100C_disk"])
def test_emulated_shards_spill_and_merge_to_golden(name, world, built, workdir, files):
    """Every shard spills at least once; some insert_keys call hands a shard more keys that cannot all find a slot than the
    failure list holds (2 groups and a deferred list: 3 groups at most), which only works when the call is cut into slices
    of one group with a spill between them; the merged shards, concatenated, are the golden."""
    args, ins, g = CASES[name]
    out = os.path.join(workdir, "dme_%s_%d" % (name, world))
    h, b, spills, sh = _emulate(args, [files[i] for i in ins], world, out)
    assert min(spills) >= 1, spills
    assert sh.most_failing > 3 * sh.fail_group, (sh.most_failing, sh.fail_group)
    _check(h, b, g)


def test_emulated_shards_quality_filter_matches_count_disk(built, workdir, inputs):
    """-Q on the golden_qual reads: the same bytes as the single-GPU count --disk of the same switches."""
    args, ins = QUAL_CASES["q_fq"]
    args = [a if a != "1M" else "8k" for a in args] + ["--disk"]
    paths = [inputs[i] for i in ins]
    ref = _one_gpu("count", args, os.path.join(workdir, "dmq_ref.jf"), paths)
    for world in (2, 4):
        h, b, spills, _ = _emulate(args, paths, world, os.path.join(workdir, "dmq_%d" % world), chunk=60000)
        assert min(spills) >= 1 and b == ref, (world, spills)


def test_emulated_shards_owner_bloom_filter_survives_spills(built, workdir, inputs):
    """--bf-size on the owner (the filter is not the table: a spill does not clear it), on input whose k-mers mostly occur
    twice, so that the shards fill: every k-mer seen at least twice is counted once less or exactly (the prefilter's
    contract, test_gpu_shard_bloom.py), none more often, and no k-mer that is not in the input appears.  The occurrences
    are the single-GPU count --disk of the same switches without the filter."""
    args = ["-m", "21", "-s", "100k", "-C", "--disk"]
    paths = [inputs[i] for i in ("plain.fa", "multi.fa", "plain.fa")]
    ref = os.path.join(workdir, "dmb_ref.jf")
    _one_gpu("count", args, ref, paths)
    occ = dict(jfutil.records(*jfutil.split_db(ref)))
    for world in (2, 4):
        h, b, spills, _ = _emulate(args + ["--bf-size", "1M"], paths, world, os.path.join(workdir, "dmb_%d" % world))
        assert min(spills) >= 1, spills
        got = dict(jfutil.records(h, b))
        assert set(got) <= set(occ)
        assert all(got.get(key, 0) in (n - 1, n) for key, n in occ.items() if n >= 2)
        assert all(v <= occ[key] for key, v in got.items())


def test_hash_counter_set_spill(built, workdir, inputs):
    """HashCounter.set_spill from Python (one GPU, no doubling): the pieces merged are the golden; a hook that raises ends
    the count with JellyfishError ERR_SINK, the exception named in its message."""
    from jellyfish_b200 import HashCounter, JellyfishError, _lib
    from jellyfish_b200.distributed import DiskPieces
    args, ins, g = CASES["disk_k21_LU"]
    size, eng, (lo, hi), ocl = _opts(args)
    out = os.path.join(workdir, "dmhc.jf")
    with HashCounter(size, eng.pop("val_len"), allow_regrow=False, **eng) as hc:
        dp = DiskPieces(hc, out, 0, ocl)
        hc.add_files([inputs[i] for i in ins])
        hc.done()
        assert len(dp.pieces) >= 1
        dp.write_output(out + ".0", lo, hi)
    _check(*jfutil.split_db(out + ".0"), g)

    def bad(hc):
        raise OSError("disk full")
    with HashCounter(size, 7, allow_regrow=False, **eng) as hc:
        hc.set_spill(bad)
        with pytest.raises(JellyfishError) as ex:
            hc.add_files([inputs[i] for i in ins])
            hc.done()
        assert ex.value.code == _lib.ERR_SINK and "disk full" in str(ex.value)


def _torchrun(world, extra, args, out, paths, port):
    env = dict(os.environ, SOURCE_DATE_EPOCH="0")
    for v in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        env.pop(v, None)
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(world), "--master-addr",
                        "127.0.0.1", "--master-port", str(port), os.path.join(HERE, "disk_ranks_worker.py"), json.dumps(extra)]
                       + args + ["-o", out] + paths, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, timeout=900, cwd=jfutil.ROOT, env=env)
    log = r.stdout.decode(errors="replace")
    assert r.returncode == 0, log[-3000:]
    return jfutil.split_db(out), log


@pytest.mark.skipif(_ngpu() < 2, reason="needs at least 2 GPUs")
@pytest.mark.parametrize("world", [2, 4, 8])
def test_count_multi_disk_under_torchrun(world, built, workdir, files):
    """The disk goldens through the key exchange; k = 17 on 8 Mbp with -s 2M through the record exchange (small shards
    filled region by region), against the single-GPU count --disk; a FASTQ file whose cut check fails, whose abandoned pass
    must leave no piece behind."""
    if _ngpu() < world:
        pytest.skip("needs %d GPUs" % world)
    port = 29950 + 10 * world
    for j, name in enumerate(sorted(CASES)):
        args, ins, g = CASES[name]
        out = os.path.join(workdir, "dmt_%d_%s.jf" % (world, name))
        (h, b), log = _torchrun(world, {}, args + ["--disk"], out, [files[i] for i in ins], port + j % 5)
        _check(h, b, g)
        assert "spills" in log
    fa = os.path.join(workdir, "dmt_8m.fa")
    if not os.path.exists(fa):
        gen.generate_sequence_fasta(fa, 7, 8000000)
    args = ["-m", "17", "-s", "2M", "-C", "--disk"]
    ref = _one_gpu("count", args, os.path.join(workdir, "dmt_8m_ref.jf"), [fa])
    (h, b), log = _torchrun(world, {"part_min_mb": 1, "pool_bytes": 4 << 30}, args, os.path.join(workdir, "dmt_%d_8m.jf" % world), [fa], port + 6)
    assert "EXCHANGE rank 0 records" in log, log[-3000:]
    spills = [int(x.split()[0]) for x in log.split("--disk: spills ")[1:]]
    assert len(spills) == world and min(spills) >= 1, spills
    assert b == ref
    fq = os.path.join(workdir, "dmt_fooled_%d.fq" % world)
    with open(fq, "wb") as f:
        f.write(_fooled_fastq(world, 21))
    args = ["-m", "21", "-s", "4k", "-C", "--disk"]
    ref = _one_gpu("count", args, os.path.join(workdir, "dmt_fq_ref.jf"), [fq])
    out = os.path.join(workdir, "dmt_%d_fq.jf" % world)
    (h, b), log = _torchrun(world, {}, args, out, [fq], port + 7)
    assert "counting whole files per rank instead" in log and b == ref
    assert not [f for f in os.listdir(workdir) if f.startswith(os.path.basename(out) + ".")]
