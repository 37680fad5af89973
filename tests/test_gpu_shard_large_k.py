"""Sharded counting of k-mers longer than 64 bases (four-word keys): the k-mers are bucketed by the shard that owns their
table position (jfgpu_extract_route), inserted by their owner (jfgpu_insert_keys), and the rank-ordered concatenation of
the shard dumps equals the reference's database byte for byte (tests/golden/golden_large_k.json).  Most tests run every
shard's engine on one device, the data path of the multi-GPU command without NCCL; the torchrun test needs >= 2 GPUs."""
import collections
import json
import os
import random
import subprocess
import sys

import pytest

import gen
import jfutil

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = json.load(open(os.path.join(HERE, "golden", "golden_large_k.json")))
# the golden cases that neither double nor need --if, --disk or --text
CASES = ["k65", "k65C_multi_files", "k72_Q_quality", "k96C_dos", "k96_noeol_lower", "k100C_LU", "k100C_Q", "k100C_fastq",
         "k100C_long_header", "k100C_ocl1", "k100_one_per_line", "k128C", "k128_multi"]
UINT64_MAX = (1 << 64) - 1


def _ngpu():
    try:
        import torch
        return torch.cuda.device_count()
    except Exception:
        return 0


def _size(v):
    return int(v[:-1]) * {"k": 10**3, "M": 10**6, "G": 10**9}[v[-1]] if v[-1] in "kMG" else int(v)


def _opts(args):
    """-> (engine keyword arguments, dump keyword arguments) of a golden case's count switches"""
    rest = [a for a in args if a != "-C"]
    o = dict(zip(rest[0::2], rest[1::2]))
    eng = {"k": int(o["-m"]), "canonical": "-C" in args}
    if "-Q" in o:
        eng["min_qual"] = o["-Q"]
    if "--min-quality" in o:
        eng["min_qual"] = int(o.get("--quality-start", 64)) + int(o["--min-quality"])
    dump = {"lower": int(o.get("-L", 0)), "upper": int(o.get("-U", UINT64_MAX)), "out_counter_len": int(o.get("--out-counter-len", 4))}
    return _size(o["-s"]), eng, dump


def _cuts(data, chunk, fastq_records):
    """Offsets that cut `data` into pieces of about `chunk` bytes.  No piece but the last ends on '\\r' (the parser looks one
    byte past it); with `fastq_records` every piece ends behind a complete 4-line record (-Q reads the quality line two lines
    below the bases)."""
    if fastq_records:
        ends, lines = [], 0
        for i, c in enumerate(data):
            if c == 10:
                lines += 1
                if lines % 4 == 0:
                    ends.append(i + 1)
        cuts, last = [], 0
        for e in ends:
            if e - last >= chunk and e < len(data):
                cuts.append(e)
                last = e
        return cuts
    cuts = []
    off = chunk
    while off < len(data):
        c = off
        while c > 1 and data[c - 1] == 13:
            c -= 1
        cuts.append(c)
        off = c + chunk
    return cuts


class Shards(object):
    """`world` engines of one global table on the current device, fed through extract_route / insert_keys."""

    def __init__(self, size, world, cap=1 << 20, **eng):
        import torch
        from jellyfish_b200 import HashCounter
        self.world = world
        self.hcs = [HashCounter(size, 7, shard_index=r, n_shards=world, allow_regrow=False, max_batch_bytes=1 << 20, **eng)
                    for r in range(world)]
        assert self.hcs[0].key_words == 4
        self.cap = cap
        self.keys = torch.zeros((world, cap * 4), dtype=torch.int64, device="cuda")
        self.counts = torch.zeros(world, dtype=torch.int64, device="cuda")
        self.routed = 0
        self.handed = [0] * world
        self.n_files = 0

    def add(self, data, chunk=60000, fastq_records=False):
        import torch
        router = self.hcs[self.n_files % self.world]      # any shard can route: every shard has the same matrix
        self.n_files += 1
        bounds = [0] + _cuts(data, chunk, fastq_records) + [len(data)]
        for a, b in zip(bounds[:-1], bounds[1:]):
            # every piece in a buffer of its own: device text starts 16-byte aligned, and a call reads nothing outside it
            buf = torch.zeros(b - a + 256, dtype=torch.uint8, device="cuda")
            if b > a:
                buf[:b - a] = torch.frombuffer(bytearray(data[a:b]), dtype=torch.uint8).cuda()
            self.counts.zero_()
            torch.cuda.synchronize()
            router.extract_route(buf.data_ptr(), b - a, self.keys.data_ptr(), self.cap, self.counts.data_ptr(),
                                 begin=a == 0, end=b >= len(data))
            c = self.counts.tolist()
            assert max(c) <= self.cap
            for d in range(self.world):
                self.hcs[d].insert_keys(self.keys[d].data_ptr(), c[d])
                self.handed[d] += c[d]
            self.routed += sum(c)

    def dump(self, out, **dump):
        from jellyfish_b200.distributed import concat_shards
        stats = []
        for r, hc in enumerate(self.hcs):
            stats.append(hc.done())
            hc.dump("%s.%d" % (out, r), **dump)
        return stats, jfutil.split_db(concat_shards(out, self.world, out + ".jf"))

    def close(self):
        for hc in self.hcs:
            hc.close()


@pytest.mark.parametrize("world", [2, 4, 8])
@pytest.mark.parametrize("name", CASES)
def test_sharded_case_against_reference_golden(name, world, built, workdir, inputs):
    g = GOLDEN["cases"][name]
    size, eng, dump = _opts(g["args"])
    sh = Shards(size, world, cap=200000, **eng)
    try:
        for f in g["inputs"]:
            data = open(inputs[f], "rb").read()
            sh.add(data, fastq_records="min_qual" in eng and data[:1] == b"@")
        stats, (h, b) = sh.dump(os.path.join(workdir, "shk_%s_%d" % (name, world)), **dump)
    finally:
        sh.close()
    assert sum(s["inserted"] for s in stats) == sh.routed
    assert sum(s["kmers"] for s in stats) == sh.routed
    assert [s["inserted"] for s in stats] == sh.handed
    assert jfutil.semantic(h) == g["header"]
    assert jfutil.md5(b) == g["body_md5"]


def test_sharded_large_key_sh_s2M(built, workdir):
    """The reference's large_key.sh (k = 100, -s 2M) over 4 shards"""
    p = os.path.join(workdir, "shard_seq1m_0_10001.fa")
    gen.generate_sequence_fasta(p + ".full", 1040104553, 1000000)
    with open(p + ".full", "rb") as f:
        lines = f.read().split(b"\n")
    data = b"\n".join(lines[:10001]) + b"\n"
    g = GOLDEN["large_key"]["s2M"]
    sh = Shards(_size(g["args"][g["args"].index("-s") + 1]), 4, cap=400000, k=100)
    try:
        sh.add(data, chunk=250000)
        stats, (h, b) = sh.dump(os.path.join(workdir, "shk_large_key"))
    finally:
        sh.close()
    assert sum(s["inserted"] for s in stats) == sh.routed
    db = os.path.join(workdir, "shk_large_key.jf")
    out = jfutil.run([jfutil.OUR_JF, "dump", "-c", db]).stdout
    mers = b"".join(sorted(line.split(b" ")[0] + b"\n" for line in out.splitlines()))
    assert jfutil.md5(mers) == g["sorted_mers_md5"] == "ded3925fe6bbaca10accc10d1bde11b5"
    assert jfutil.semantic(h) == g["header"]
    assert jfutil.md5(b) == g["body_md5"]


def _model(seq, k, canonical=True):
    """count of every canonical k-mer of a sequence without resets, with Python ints"""
    code = {65: 0, 67: 1, 71: 2, 84: 3}
    mask = (1 << (2 * k)) - 1
    f = r = 0
    out = collections.Counter()
    for i, ch in enumerate(seq):
        c = code[ch]
        f = ((f << 2) | c) & mask
        r = (r >> 2) | ((3 - c) << (2 * (k - 1)))
        if i >= k - 1:
            out[min(f, r) if canonical else f] += 1
    return out


def test_sharded_hot_keys_period3_and_polya(built, workdir):
    """Every k-mer of the text is one of three (period-3 repeat) or one (poly-A) keys: the route buckets of one to three
    owners take all of them, and the owners' claim / publish inserts run under full contention."""
    for unit, n in ((b"ACG", 3000000), (b"A", 2000000)):
        seq = (unit * (n // len(unit) + 1))[:n]
        model = _model(seq, 100)
        sh = Shards(1 << 12, 4, cap=1 << 20, k=100, canonical=True)
        try:
            sh.add(gen.fasta(seq), chunk=1000000)
            stats, (h, b) = sh.dump(os.path.join(workdir, "shk_hot"))
        finally:
            sh.close()
        assert sum(s["kmers"] for s in stats) == n - 99 == sh.routed
        assert 1 <= sum(1 for c in sh.handed if c) <= len(model) <= 3
        assert dict(jfutil.records(h, b)) == dict(model)


def test_sharded_lookup_histogram_and_dump_against_model(built, workdir):
    """get_many on every shard: the owner of a key gives its count, every other shard 0; histograms add up over the
    shards; the concatenated dump is the model."""
    seq = gen._seq(600000, 91)
    seq = seq[:500000] + seq[100000:300000]             # repeated stretch: counts of 2
    model = _model(seq, 100)
    world = 4
    sh = Shards(1 << 21, world, cap=400000, k=100, canonical=True)
    try:
        sh.add(gen.fasta(seq), chunk=200000)
        stats, (h, b) = sh.dump(os.path.join(workdir, "shk_model"))
        assert dict(jfutil.records(h, b)) == dict(model)
        assert sum(s["distinct"] for s in stats) == len(model)
        rng = random.Random(7)
        sample = rng.sample(sorted(model), 2000) + [rng.getrandbits(200) for _ in range(50)]
        lsize = h["size"].bit_length() - 1
        got = [hc.get_many(sample) for hc in sh.hcs]
        for i, key in enumerate(sample):
            owner = jfutil.hash_pos(h, key) >> (lsize - 2)
            for r in range(world):
                assert got[r][i] == (model.get(key, 0) if r == owner else 0), (i, r, owner)
        assert [sum(got[r][i] for r in range(world)) for i in range(len(sample))] == [model.get(x, 0) for x in sample]
        hists = [hc.histogram(4) for hc in sh.hcs]
        want = collections.Counter(min(v, 3) for v in model.values())
        assert [sum(hh[c] for hh in hists) for c in (1, 2, 3)] == [want[1], want[2], want[3]]
    finally:
        sh.close()


def test_sharded_full_shard_raises_hash_full(built, workdir):
    """A shard too small for the keys it owns fails with "Hash full" (JFGPU_ERR_FULL): no doubling across shards, no spill,
    and no key is dropped silently."""
    from jellyfish_b200 import JellyfishError
    from jellyfish_b200 import _lib as L
    seq = gen._seq(100000, 92)
    sh = Shards(1 << 10, 2, cap=200000, k=100, canonical=True)
    try:
        sh.add(gen.fasta(seq))
        for r, hc in enumerate(sh.hcs):
            with pytest.raises(JellyfishError) as ei:
                hc.done()
            assert ei.value.code == L.ERR_FULL
            st = hc.stats()
            assert st["distinct"] <= hc.info()["local_slots"]
            assert st["inserted"] <= sh.handed[r]
            assert st["inserted"] < sh.handed[r]
        assert sum(sh.handed) == sh.routed == len(seq) - 99
    finally:
        sh.close()


@pytest.mark.skipif(_ngpu() < 2, reason="needs at least 2 GPUs")
@pytest.mark.parametrize("name,world", [("k65C_multi_files", 2), ("k128C", 2), ("k65C_multi_files", 4), ("k128C", 4),
                                        ("k65C_multi_files", 8), ("k128C", 8)])
def test_sharded_count_torchrun_matches_golden(name, world, built, workdir, inputs):
    if _ngpu() < world:
        pytest.skip("needs %d GPUs" % world)
    from jellyfish_b200.distributed import concat_shards
    g = GOLDEN["cases"][name]
    size, eng, dump = _opts(g["args"])
    out = os.path.join(workdir, "shk_multi_%s_%d" % (name, world))
    cfg = {"size": size, "k": eng["k"], "canonical": eng["canonical"], "files": [inputs[i] for i in g["inputs"]], "out": out,
           "batch_bytes": 300000}
    worker = os.path.join(HERE, "multi_worker.py")
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(world),
                        "--master-addr", "127.0.0.1", "--master-port", "29643", worker, json.dumps(cfg)],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, timeout=600, env=dict(os.environ, SOURCE_DATE_EPOCH="0"))
    assert r.returncode == 0, r.stdout.decode()[-3000:]
    assert b"exchange: keys" in r.stdout
    h, b = jfutil.split_db(concat_shards(out, world, out + ".jf"))
    assert jfutil.semantic(h) == g["header"]
    assert jfutil.md5(b) == g["body_md5"]
