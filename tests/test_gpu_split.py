"""One input file split among shards (jellyfish_b200/split.py) on one H100: one engine per shard, as the multi-GPU path
runs them, each counting its share streamed in small pieces (ShareReader) after the seam in front of it (jfgpu_seam).  The
concatenated shard dumps must be the golden databases byte for byte; Bloom counters built from the shares and folded must
be the golden counters."""
import ctypes as C
import json
import os

import numpy as np
import pytest

import jfutil
from cases import BC_CASES, CASES

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(__file__)
GOLDEN = json.load(open(os.path.join(HERE, "golden", "golden.json")))
GOLDEN_LK = json.load(open(os.path.join(HERE, "golden", "golden_large_k.json")))
GOLDEN_BC = json.load(open(os.path.join(HERE, "golden", "golden_bc.json")))
PIECE = 300000            # small pieces: cuts and piece ends fall inside the shares


def _size(v):
    return int(v[:-1]) * {"k": 10**3, "M": 10**6, "G": 10**9}[v[-1]] if v[-1] in "kMG" else int(v)


def _stream_share(hc, path, share, stage, extract, tally=None):
    """The seam, then the share's pieces copied into `stage` (device) and handed to extract(ptr, n, begin, end)."""
    import torch
    from jellyfish_b200 import _lib
    from jellyfish_b200.distributed import ShareReader
    lib = _lib.load()
    reader = ShareReader(path, share, PIECE + ShareReader.CR_SLACK)
    try:
        seam = reader.seam()
        if seam:
            t = torch.frombuffer(bytearray(seam), dtype=torch.uint8).cuda()
            hc.seam(t.data_ptr(), len(seam), fmt=share.fmt)
        for i in range(reader.n_pieces):
            hptr, n, begin, end = reader.read(i)
            assert lib.jfgpu_memcpy_h2d(C.c_void_p(stage.data_ptr()), C.c_void_p(hptr), n, None) == 0
            torch.cuda.synchronize()
            reader.release(i)
            if tally is not None:
                hc.count_newlines(stage.data_ptr(), n, tally.data_ptr())
            extract(stage.data_ptr(), n, begin, end, share.fmt)
    finally:
        reader.close()


def _key_exchange(paths, k, size, canonical, world, fastq_fail=False):
    """Every file split among `world` shard engines, keys routed with jfgpu_extract_route and inserted by their owners.
    -> the concatenated database (header, body).  fastq_fail: pretend the FASTQ check failed, clear and count whole files."""
    import torch
    from jellyfish_b200 import HashCounter, split
    shards = [HashCounter(size, 7, k=k, canonical=canonical, shard_index=r, n_shards=world, allow_regrow=False, max_batch_bytes=1 << 20)
              for r in range(world)]
    kw = shards[0].key_words
    cap = PIECE + 65536
    keys = torch.zeros((world, cap * kw), dtype=torch.int64, device="cuda")
    counts = torch.zeros(world, dtype=torch.int64, device="cuda")
    stage = torch.zeros(PIECE + (8 << 10), dtype=torch.uint8, device="cuda")

    def router(r):
        def extract(ptr, n, begin, end, fmt):
            counts.zero_()
            torch.cuda.synchronize()
            shards[r].extract_route(ptr, n, keys.data_ptr(), cap, counts.data_ptr(), begin=begin, end=end, fmt=fmt)
            c = counts.tolist()
            for d in range(world):
                shards[d].insert_keys(keys[d].data_ptr(), c[d])
            torch.cuda.synchronize()
        return extract

    tallies = []
    for path in paths:
        shares = [split.plan_file(path, r, world, k) for r in range(world)]
        if shares[0] is None:
            continue
        fq = []
        for r, sh in enumerate(shares):
            tally = torch.zeros(1, dtype=torch.int64, device="cuda")
            _stream_share(shards[r], path, sh, stage, router(r), tally)
            fq.append((sh.end - sh.start, int(tally.item())))
        if sh.fmt == "fastq":
            tallies.append(fq)
            data = open(path, "rb").read()
            assert fq == [(s.end - s.start, data[s.start:s.end].count(b"\n")) for s in shares]
    # the golden FASTQ inputs are cut on records: the check must pass (only fastq_fail takes the whole-file path)
    assert all(split.fastq_cuts_ok(t) for t in tallies)
    if fastq_fail:
        for hc in shards:
            hc.clear()
        for i, path in enumerate(paths):
            data = open(path, "rb").read()
            buf = torch.zeros(len(data) + 256, dtype=torch.uint8, device="cuda")
            if data:
                buf[:len(data)] = torch.frombuffer(bytearray(data), dtype=torch.uint8).cuda()
            for off in range(0, len(data), PIECE):
                ln = min(PIECE, len(data) - off)
                stage[:ln].copy_(buf[off:off + ln])
                router(i % world)(stage.data_ptr(), ln, off == 0, off + ln >= len(data), None)
    return _dump(shards, world)


def _dump(shards, world):
    from jellyfish_b200.distributed import concat_shards
    import tempfile
    with tempfile.TemporaryDirectory() as d:
        out = os.path.join(d, "split")
        for r, hc in enumerate(shards):
            hc.done()
            hc.dump("%s.%d" % (out, r))
            hc.close()
        return jfutil.split_db(concat_shards(out, world, out + ".jf"))


def _case(name):
    if name in CASES:
        return CASES[name][0], CASES[name][1], GOLDEN[name]
    c = GOLDEN_LK["cases"][name]
    return c["args"], c["inputs"], c


KEY_CASES = ["k31C", "multi", "long_header", "one_per_line", "blank_runs", "fq", "k63C", "k63_multi", "k100C_long_header",
             "k100C_fastq", "k65C_multi_files", "k100_one_per_line"]


@pytest.mark.parametrize("world", [2, 4, 8])
@pytest.mark.parametrize("name", KEY_CASES)
def test_split_key_exchange(name, world, built, inputs):
    args, ins, g = _case(name)
    k = int(args[args.index("-m") + 1])
    h, b = _key_exchange([inputs[f] for f in ins], k, _size(args[args.index("-s") + 1]), "-C" in args, world)
    assert jfutil.semantic(h) == g["header"]
    assert jfutil.md5(b) == g["body_md5"]


def test_fastq_fallback_counts_whole_files(built, inputs):
    args, ins, g = _case("fq")
    h, b = _key_exchange([inputs[f] for f in ins], 21, _size("1M"), True, 4, fastq_fail=True)
    assert jfutil.md5(b) == g["body_md5"]


@pytest.mark.parametrize("name,world", [("multi_files", 2), ("multi_files", 4), ("k15C", 2), ("fq_dos", 2), ("c3", 2), ("x17_4M", 8)])
def test_split_record_exchange(name, world, built, inputs):
    """k <= 21: the record exchange (jfgpu_shard_extract / _pack / _unpack), chunks copied the way the all-to-all moves them.
    (The geometries and worlds of tests/test_gpu_parity.py::test_record_exchange_on_one_gpu that have a golden database: the
    record form needs regions of a table of at least a few hundred thousand slots per shard.)"""
    import torch
    from jellyfish_b200 import HashCounter, split
    from jellyfish_b200.distributed import CHUNK
    # (x17_4M: eight shards need a table of 4M slots to be filled region by region and no golden has that size; the
    # yardstick is the single-GPU engine, itself held to the goldens)
    args, ins, g = _case(name) if name != "x17_4M" else (["-m", "17", "-s", "4M", "-C"], ["plain1m.fa"], None)
    k = int(args[args.index("-m") + 1])
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    arena = 2 * n_sm * max(1, 1024 // world) + 64
    torch.cuda.empty_cache()
    shards, bufs = [], []
    for r in range(world):
        hc = HashCounter(_size(args[args.index("-s") + 1]), int(args[args.index("-c") + 1]) if "-c" in args else 7, k=k, canonical="-C" in args, shard_index=r, n_shards=world,
                         allow_regrow=False, part_min_mb=1, pool_bytes=2 << 30, max_batch_bytes=1 << 20)
        bb = [torch.empty(2 * world * arena * CHUNK, dtype=torch.uint8, device="cuda"), torch.empty(2 * world * arena * 8, dtype=torch.uint8, device="cuda"),
              torch.empty(world * arena * CHUNK, dtype=torch.uint8, device="cuda"), torch.empty(world * arena * 8, dtype=torch.uint8, device="cuda")]
        assert hc.shard_setup(bb[0].data_ptr(), bb[1].data_ptr(), arena, bb[2].data_ptr(), bb[3].data_ptr(), arena)
        shards.append(hc)
        bufs.append(bb)
    stage = torch.zeros(PIECE + (8 << 10), dtype=torch.uint8, device="cuda")
    n_round = [0]

    def sender(src):
        def extract(ptr, n, begin, end, fmt):
            bank = n_round[0] & 1
            n_round[0] += 1
            shards[src].shard_extract(ptr, n, bank, begin=begin, end=end, fmt=fmt)
            counts = shards[src].shard_pack(bank)
            send, send_dir = bufs[src][0], bufs[src][1]
            for d in range(world):
                c = counts[d]
                recv, recv_dir = bufs[d][2], bufs[d][3]
                a0 = (bank * world + d) * arena
                recv[src * arena * CHUNK:(src * arena + c) * CHUNK] = send[a0 * CHUNK:(a0 + c) * CHUNK]
                recv_dir[src * arena * 8:(src * arena + c) * 8] = send_dir[a0 * 8:(a0 + c) * 8]
                torch.cuda.synchronize()
                got = [0] * world
                got[src] = c
                shards[d].shard_unpack(got)
                torch.cuda.synchronize()
        return extract

    for f in ins:
        for r in range(world):
            sh = split.plan_file(inputs[f], r, world, k)
            if sh is not None:
                _stream_share(shards[r], inputs[f], sh, stage, sender(r))
    h, b = _dump(shards, world)
    del shards, bufs
    if g is None:
        torch.cuda.empty_cache()
        with HashCounter(_size(args[args.index("-s") + 1]), 7, k=k, canonical=True) as one:
            one.add_files([inputs[f] for f in ins])
            one.done()
            assert b == one.dump_records()
        return
    assert jfutil.semantic(h) == g["header"]
    assert jfutil.md5(b) == g["body_md5"]


@pytest.mark.parametrize("world", [2, 4, 8])
@pytest.mark.parametrize("name", ["bc_k21C", "bc_k63C"])
def test_split_bloom_counter(name, world, built, inputs):
    """`bc` across ranks: a counter per share (jfgpu_seam_host, then host feeds with the format flag), folded into one."""
    import torch
    from jellyfish_b200 import split
    from jellyfish_b200.engine import BloomCounter
    from jellyfish_b200.distributed import ShareReader
    bargs, bins, _, _ = BC_CASES[name]
    k = int(bargs[bargs.index("-m") + 1])
    size = _size(bargs[bargs.index("-s") + 1])
    fpr = float(bargs[bargs.index("-f") + 1]) if "-f" in bargs else 0.001
    parts = [BloomCounter(size, fpr, k=k, canonical="-C" in bargs) for _ in range(world)]
    for f in bins:
        for r in range(world):
            sh = split.plan_file(inputs[f], r, world, k)
            if sh is None:
                continue
            reader = ShareReader(inputs[f], sh, PIECE + ShareReader.CR_SLACK)
            seam = reader.seam()
            if seam:
                parts[r].seam_text(seam, fmt=sh.fmt)
            for i in range(reader.n_pieces):
                hptr, n, begin, end = reader.read(i)
                parts[r].add_text((hptr, n), begin=begin, end=end, fmt=sh.fmt)
                reader.release(i)
            reader.close()
    words0, n_words = parts[0].words()
    for p in parts[1:]:
        ptr, n = p.words()
        assert n == n_words
        parts[0].fold(ptr, 0, n)
    torch.cuda.synchronize()
    chunks = []
    parts[0].dump_range(0, parts[0].info()["nb_bytes"], chunks.append)
    for p in parts:
        p.close()
    assert jfutil.md5(b"".join(chunks)) == GOLDEN_BC[name]["bc_md5"]


@pytest.mark.parametrize("k", [21, 31, 100])
def test_seam_then_feed_equals_one_feed(k, built, inputs):
    """jfgpu_seam over [c, s) then a continuation feed of [s, S) counts what a feed of [0, S) counts of the k-mers ending in
    [s, S): the database of [0, s) fed whole plus [s, S) after the seam is the database of the whole file."""
    import torch
    from jellyfish_b200 import HashCounter, split
    data = open(inputs["multi.fa"], "rb").read()
    rd = lambda off, n: data[off:off + n]
    bodies = []
    for how in ("whole", "device", "host"):
        with HashCounter(1 << 20, 7, k=k, canonical=True) as hc:
            if how == "whole":
                hc.add_text(data)
            else:
                cuts = [0] + [split.share_start(rd, len(data), "fasta", a) for a in (len(data) // 3, 2 * len(data) // 3)] + [len(data)]
                for s, e in zip(cuts, cuts[1:]):
                    c = split.fasta_seam_start(rd, s, k)
                    if how == "host":
                        if c < s:
                            hc.seam_text(data[c:s], fmt="fasta")
                        hc.add_text(data[s:e], begin=c >= s, end=True, fmt="fasta")
                    else:
                        if c < s:
                            t = torch.frombuffer(bytearray(data[c:s]), dtype=torch.uint8).cuda()
                            hc.seam(t.data_ptr(), s - c, fmt="fasta")
                        t = torch.zeros(e - s + 256, dtype=torch.uint8, device="cuda")
                        t[:e - s] = torch.frombuffer(bytearray(data[s:e]), dtype=torch.uint8).cuda()
                        hc.add_device_text(t.data_ptr(), e - s, begin=c >= s, end=True, fmt="fasta")
            st = hc.done()
            bodies.append((hc.dump_records(), st["kmers"]))
    assert bodies[1] == bodies[0] and bodies[2] == bodies[0]


def test_seam_counts_nothing_and_refuses_qual(built):
    from jellyfish_b200 import HashCounter, JellyfishError
    with HashCounter(1 << 16, 7, k=21) as hc:
        hc.seam_text(b">x\n" + b"ACGT" * 100 + b"\n")
        assert hc.stats()["kmers"] == 0
        assert hc.done()["distinct"] == 0
    with HashCounter(1 << 16, 7, k=21, min_qual="5") as hc:
        with pytest.raises(JellyfishError):
            hc.seam_text(b">x\nACGT\n")


def test_count_newlines_against_numpy(built):
    import torch
    from jellyfish_b200 import HashCounter
    rng = np.random.default_rng(5)
    text = rng.choice(np.frombuffer(b"ACGT\n\r>", np.uint8), 1 << 20).astype(np.uint8)
    dev = torch.from_numpy(text).cuda()
    cnt = torch.zeros(1, dtype=torch.int64, device="cuda")
    with HashCounter(1 << 16, 7, k=21) as hc:
        for off, n in [(0, 0), (0, 1), (1, 15), (3, 16), (7, 17), (15, 4097), (0, 1 << 20), (9, (1 << 20) - 9), (13, 123457)]:
            cnt.zero_()
            hc.count_newlines(dev.data_ptr() + off, n, cnt.data_ptr())
            torch.cuda.synchronize()
            assert int(cnt.item()) == int(np.count_nonzero(text[off:off + n] == 10)), (off, n)
