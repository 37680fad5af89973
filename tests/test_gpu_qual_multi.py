"""-Q and --if across shards on one H100: one engine per shard, as `count_multi` runs them, FASTQ text cut behind whole
records (jfgpu_fastq_cuts for device text, ShareReader(records=True) for the pieces of a share) and FASTA split at header
lines.  The concatenated shard dumps must be the golden databases byte for byte; the cut kernel is held to a numpy model,
and cuts aimed at every byte of one read to the text model (tests/text_model.py)."""
import bisect
import ctypes as C
import json
import os
import random

import numpy as np
import pytest

import jfutil
import text_model as tm
from cases import CASES, QUAL_CASES

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(__file__)
GOLDEN = json.load(open(os.path.join(HERE, "golden", "golden.json")))
GOLDEN_QUAL = json.load(open(os.path.join(HERE, "golden", "golden_qual.json")))
PIECE = 60000             # small pieces of a share, so that piece ends fall inside the files and inside FASTQ records
PIECE_LONG = 400000       # reads_long.fq: the record slack (a quarter of a piece) must hold its 80 KB reads
ROUND = 150000            # rounds of a whole file in device memory
NAMES = sorted(n for n in QUAL_CASES if n not in ("q_ml", "q_mixed")) + ["if_sub", "if_zeros", "if_k40_rep"]


def _size(v):
    return int(v[:-1]) * {"k": 10**3, "M": 10**6, "G": 10**9}[v[-1]] if v[-1] in "kMG" else int(v)


def _case(name, inputs):
    """-> (engine arguments, --if paths, input paths, golden)"""
    args, ins = (CASES[name] if name in CASES else QUAL_CASES[name])
    g = GOLDEN[name] if name in CASES else GOLDEN_QUAL[name]
    o, ifs, i = {}, [], 0
    while i < len(args):
        a = args[i]
        if a == "-C":
            o["-C"] = True
            i += 1
            continue
        if a == "--if":
            ifs.append(inputs[args[i + 1][1:]])
        else:
            o[a] = args[i + 1]
        i += 2
    eng = {"k": int(o["-m"]), "canonical": "-C" in o, "size": _size(o["-s"])}
    if "-Q" in o:
        eng["min_qual"] = ord(o["-Q"])
    if "--min-quality" in o:
        eng["min_qual"] = int(o.get("--quality-start", 64)) + int(o["--min-quality"])
    return eng, ifs, [inputs[f] for f in ins], g


@pytest.fixture(scope="module")
def cuda(built):
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return torch


def _dev(torch, data, pad=256):
    t = torch.zeros(len(data) + pad, dtype=torch.uint8, device="cuda")
    if len(data):
        t[:len(data)] = torch.frombuffer(bytearray(data), dtype=torch.uint8).cuda()
    return t


# ---- the cut kernel against a model ---------------------------------------------------------------------------------

def _model_cuts(data, target, phase):
    nl = np.flatnonzero(np.frombuffer(data, np.uint8) == 10)
    idx = phase + 1 + np.arange(len(nl))
    ends = list(nl[idx % 4 == 0] + 1)
    cuts, o = [], 0
    while o + target < len(data):
        j = bisect.bisect_right(ends, o + target) - 1
        if j < 0 or ends[j] <= o:
            return None, (phase + len(nl)) % 4
        cuts.append(int(ends[j]))
        o = cuts[-1]
    return cuts, (phase + len(nl)) % 4


def _fastq(rng, n_reads, eol=b"\n", longest=400):
    out = []
    for i in range(n_reads):
        ln = rng.randrange(0, longest)
        out.append(b"@r%d" % i + eol + bytes(rng.choice(b"ACGT") for _ in range(ln)) + eol + b"+" + eol + b"I" * ln + eol)
    return b"".join(out)


def test_fastq_cuts_match_the_model(cuda):
    torch = cuda
    from jellyfish_b200 import HashCounter, JellyfishError
    from jellyfish_b200 import _lib as L
    rng = random.Random(7)
    texts = [_fastq(rng, 3000), _fastq(rng, 2000, eol=b"\r\n"), _fastq(rng, 30, longest=5000)[:-1], b"",
             bytes(rng.choice(b"\n\nAC@+") for _ in range(200000))]        # (any text: the rule only counts lines)
    with HashCounter(1 << 16, 7, k=21, min_qual="5") as hc:
        for t, data in enumerate(texts):
            dev = _dev(torch, data)
            targets = [1, 2, 17, 1000, 16383, 16384, 16385, 50000, 123457, len(data), len(data) + 5] if data else [1, 9]
            for target in targets:
                for phase in range(4):
                    want, end = _model_cuts(data, target, phase)
                    if want is None:
                        with pytest.raises(JellyfishError) as ex:
                            hc.fastq_cuts(dev.data_ptr(), len(data), target, phase)
                        assert ex.value.code == L.ERR_FORMAT and "does not end within" in str(ex.value)
                        continue
                    got = hc.fastq_cuts(dev.data_ptr(), len(data), target, phase)
                    assert got == (want, end), (t, target, phase)
        # texts of more than 1024 tiles (16 MB): a thread of the resolving CTA then walks several tiles, and with sparse
        # lines the last record end in front of a tile comes from tiles (and threads) far back
        nprs = np.random.default_rng(11)
        for size, p_nl, targets in ((40 << 20, 1 / 50, [1000, 3000000, 700 * 16384 + 3]), (20 << 20, 1 / 30000, [200000, 1 << 20])):
            text = np.where(nprs.random(size) < p_nl, 10, nprs.choice(np.frombuffer(b"ACGT@+", np.uint8), size)).astype(np.uint8)
            data = text.tobytes()
            dev = torch.zeros(size + 256, dtype=torch.uint8, device="cuda")
            dev[:size] = torch.from_numpy(text).cuda()
            for target in targets:
                for phase in range(4):
                    want, end = _model_cuts(data, target, phase)
                    if want is None:
                        with pytest.raises(JellyfishError):
                            hc.fastq_cuts(dev.data_ptr(), size, target, phase)
                    else:
                        assert hc.fastq_cuts(dev.data_ptr(), size, target, phase) == (want, end), (size, target, phase)
            del dev
        # a record ending exactly on the target, one byte past it, and no record before the target
        rec = b"@a\nACGT\n+\nIIII\n"
        data = rec * 5
        dev = _dev(torch, data)
        assert hc.fastq_cuts(dev.data_ptr(), len(data), len(rec), 0) == ([len(rec) * i for i in range(1, 5)], 0)
        assert hc.fastq_cuts(dev.data_ptr(), len(data), len(rec) + 1, 0) == ([len(rec) * i for i in range(1, 5)], 0)
        with pytest.raises(JellyfishError):
            hc.fastq_cuts(dev.data_ptr(), len(data), len(rec) - 1, 0)
        # an oversized record in a text of many tiles
        big = _fastq(rng, 1000) + b"@big\n" + b"A" * 70000 + b"\n+\n" + b"I" * 70000 + b"\n" + _fastq(rng, 1000)
        dev = _dev(torch, big)
        with pytest.raises(JellyfishError, match="does not end within 100000 bytes"):
            hc.fastq_cuts(dev.data_ptr(), len(big), 100000, 0)
        assert hc.fastq_cuts(dev.data_ptr(), len(big), 200000, 0) == _model_cuts(big, 200000, 0)


# ---- emulated shards against the goldens ----------------------------------------------------------------------------

class _Shards(object):
    """`world` shard engines; text of rank r is routed by shard r and inserted by the owners, through the key exchange
    (extract_route / insert_keys) or the record exchange (shard_extract / _pack / _unpack, chunks copied the way the
    all-to-all moves them)."""

    def __init__(self, torch, eng, world, records):
        from jellyfish_b200 import HashCounter
        from jellyfish_b200.distributed import CHUNK
        self.torch, self.world, self.records = torch, world, records
        kw = dict(k=eng["k"], canonical=eng["canonical"], min_qual=eng.get("min_qual", 0), n_shards=world,
                  allow_regrow=False, max_batch_bytes=1 << 20)
        if records:
            kw.update(part_min_mb=1, pool_bytes=1 << 30)
        self.hc = [HashCounter(eng["size"], 7, shard_index=r, **kw) for r in range(world)]
        if records:
            n_sm = torch.cuda.get_device_properties(0).multi_processor_count
            self.arena = a = 2 * n_sm * max(1, 1024 // world) + 64
            self.bufs = []
            for hc in self.hc:
                bb = [torch.empty(2 * world * a * CHUNK, dtype=torch.uint8, device="cuda"), torch.empty(2 * world * a * 8, dtype=torch.uint8, device="cuda"),
                      torch.empty(world * a * CHUNK, dtype=torch.uint8, device="cuda"), torch.empty(world * a * 8, dtype=torch.uint8, device="cuda")]
                if not hc.shard_setup(bb[0].data_ptr(), bb[1].data_ptr(), a, bb[2].data_ptr(), bb[3].data_ptr(), a):
                    self.close()
                    pytest.skip("the record exchange does not cover this geometry")
                self.bufs.append(bb)
            self.round = 0
        else:
            self.cap = max(PIECE_LONG, ROUND) + 65536
            self.keys = torch.zeros((world, self.cap * self.hc[0].key_words), dtype=torch.int64, device="cuda")
            self.counts = torch.zeros(world, dtype=torch.int64, device="cuda")

    def extract(self, r, ptr, n, begin, end, fmt):
        torch = self.torch
        if not self.records:
            self.counts.zero_()
            torch.cuda.synchronize()
            self.hc[r].extract_route(ptr, n, self.keys.data_ptr(), self.cap, self.counts.data_ptr(), begin=begin, end=end, fmt=fmt)
            c = self.counts.tolist()
            for d in range(self.world):
                self.hc[d].insert_keys(self.keys[d].data_ptr(), c[d])
            torch.cuda.synchronize()
            return
        from jellyfish_b200.distributed import CHUNK
        bank = self.round & 1
        self.round += 1
        torch.cuda.synchronize()             # (the text may have been copied on torch's stream; the engine runs on its own)
        self.hc[r].shard_extract(ptr, n, bank, begin=begin, end=end, fmt=fmt)
        counts = self.hc[r].shard_pack(bank)
        a = self.arena
        for d in range(self.world):
            c = counts[d]
            send, send_dir = self.bufs[r][0], self.bufs[r][1]
            recv, recv_dir = self.bufs[d][2], self.bufs[d][3]
            a0 = (bank * self.world + d) * a
            recv[r * a * CHUNK:(r * a + c) * CHUNK] = send[a0 * CHUNK:(a0 + c) * CHUNK]
            recv_dir[r * a * 8:(r * a + c) * 8] = send_dir[a0 * 8:(a0 + c) * 8]
            torch.cuda.synchronize()
            got = [0] * self.world
            got[r] = c
            self.hc[d].shard_unpack(got)
            torch.cuda.synchronize()

    def set_op(self, op):
        for hc in self.hc:
            hc.set_op(op)

    def dump(self):
        from jellyfish_b200.distributed import concat_shards
        import tempfile
        with tempfile.TemporaryDirectory() as d:
            out = os.path.join(d, "q")
            for r, hc in enumerate(self.hc):
                hc.done()
                hc.dump("%s.%d" % (out, r))
            return jfutil.split_db(concat_shards(out, self.world, out + ".jf"))

    def close(self):
        for hc in self.hc:
            hc.close()
        self.hc, self.bufs = [], []


def _split_pass(sh, paths, qual, stage, piece):
    """Every file split among the shards (split.plan_file, headers under -Q) and streamed piece by piece (ShareReader).
    Returns whether every FASTQ share started on a record (split.fastq_cuts_ok of the newline tallies)."""
    from jellyfish_b200 import _lib, split
    from jellyfish_b200.distributed import ShareReader
    lib = _lib.load()
    torch = sh.torch
    ok = True
    for path in paths:
        tallies = []
        for r in range(sh.world):
            share = split.plan_file(path, r, sh.world, sh.hc[0].k, headers=qual)
            if share is None:
                continue
            reader = ShareReader(path, share, piece, records=qual and share.fmt == "fastq")
            lines = 0
            try:
                assert not reader.seam() or not qual
                seam = reader.seam()
                if seam:
                    t = _dev(torch, seam)
                    sh.hc[r].seam(t.data_ptr(), len(seam), fmt=share.fmt)
                for i in range(reader.n_pieces):
                    hptr, n, begin, end = reader.read(i)
                    reader.prefetch(i + 1)
                    assert lib.jfgpu_memcpy_h2d(C.c_void_p(stage.data_ptr()), C.c_void_p(hptr), n, None) == 0
                    torch.cuda.synchronize()
                    reader.release(i)
                    lines += C.string_at(hptr, n).count(b"\n")
                    sh.extract(r, stage.data_ptr(), n, begin, end, share.fmt)
            finally:
                reader.close()
            tallies.append((share.end - share.start, lines))
        if share.fmt == "fastq":
            ok = split.fastq_cuts_ok(tallies) and ok
    return ok


def _whole_pass(sh, paths, qual):
    """Every file read whole by rank i % world and cut into rounds (behind records for -Q FASTQ: jfgpu_fastq_cuts)."""
    from jellyfish_b200.distributed import aligned_text
    torch = sh.torch
    stage = torch.empty(max(ROUND, 1 << 20) + 256, dtype=torch.uint8, device="cuda")
    for i, path in enumerate(paths):
        data = open(path, "rb").read()
        if not data:
            continue
        r = i % sh.world
        buf = _dev(torch, data)
        if qual and data[:1] == b"@":
            cuts, _ = sh.hc[r].fastq_cuts(buf.data_ptr(), len(data), ROUND)
            bounds = [0] + cuts + [len(data)]
        else:
            bounds = list(range(0, len(data), ROUND)) + [len(data)]
        for a, b in zip(bounds, bounds[1:]):
            # (a cut behind a record starts anywhere: the extraction takes aligned text)
            sh.extract(r, aligned_text(buf.data_ptr() + a, b - a, stage), b - a, a == 0, b == len(data), None)
            torch.cuda.synchronize()


def _count(torch, eng, ifs, paths, world, records, how):
    from jellyfish_b200 import HashCounter
    qual = bool(eng.get("min_qual"))
    sh = _Shards(torch, eng, world, records)
    piece = PIECE_LONG if any(os.path.basename(p) == "reads_long.fq" for p in paths) else PIECE
    stage = torch.zeros(piece + 256, dtype=torch.uint8, device="cuda")
    try:
        def passes(run):
            ok = True
            if ifs:
                sh.set_op(HashCounter.OP_PRIME)
                ok = run(ifs) is not False
                sh.set_op(HashCounter.OP_UPDATE)
            return (run(paths) is not False) and ok
        if how == "split":
            ok = passes(lambda p: _split_pass(sh, p, qual, stage, piece))
            if not ok:                               # (count_multi's fall-back: clear, then both passes with whole files)
                for hc in sh.hc:
                    hc.clear()
                passes(lambda p: _whole_pass(sh, p, qual))
            sh.fell_back = not ok
        else:
            passes(lambda p: _whole_pass(sh, p, qual))
        return sh.dump() + (getattr(sh, "fell_back", False),)
    finally:
        sh.close()


@pytest.mark.parametrize("exchange", ["keys", "records"])
@pytest.mark.parametrize("world", [2, 4, 8])
@pytest.mark.parametrize("name", NAMES)
def test_shards_match_the_golden(name, world, exchange, cuda, inputs):
    eng, ifs, paths, g = _case(name, inputs)
    if exchange == "records" and eng["k"] > 21:
        pytest.skip("the record exchange covers k <= 21")
    for how in ("split", "whole") if world == 4 else ("split",):
        h, b, fell_back = _count(cuda, eng, ifs, paths, world, exchange == "records", how)
        assert not fell_back
        assert jfutil.semantic(h) == g["header"], how
        assert jfutil.md5(b) == g["body_md5"], how
    cuda.cuda.empty_cache()


def test_cuts_aimed_at_every_byte_of_a_read(cuda):
    """Reads with low-quality bases next to every place a cut is aimed at: round ends (jfgpu_fastq_cuts) and piece ends
    (ShareReader) at every byte of three consecutive reads, the text counted on two shards; the exact dump against the
    text model every time."""
    torch = cuda
    import tempfile
    from jellyfish_b200 import _lib, split
    from jellyfish_b200.distributed import ShareReader, aligned_text
    lib = _lib.load()
    k, q = 21, ord("5")
    rng = random.Random(3)
    recs = []
    for i in range(40):
        ln = rng.randrange(30, 90)
        qual = bytearray(rng.choice(b"IIII#") for _ in range(ln))
        recs.append(b"@r%d\n" % i + bytes(rng.choice(b"ACGT") for _ in range(ln)) + b"\n+\n" + bytes(qual) + b"\n")
    data = b"".join(recs)
    ends = [sum(len(r) for r in recs[:j]) for j in range(41)]
    aims = range(ends[19], ends[22] + 1)             # every byte of reads 19, 20 and 21
    keys, cnt, _ = tm.counts(tm.symbols(data, q), k, True)
    eng = {"k": k, "canonical": True, "size": 1 << 16, "min_qual": q}
    buf = _dev(torch, data)
    stage = torch.zeros(len(data) + 256, dtype=torch.uint8, device="cuda")
    sh = _Shards(torch, eng, 2, False)

    def check(feed, aim, what):
        for hc in sh.hc:
            hc.clear()
        feed()
        _, body = sh.dump()
        gk, gc = tm.records_to_words(body, k, 4)
        assert np.array_equal(gk, keys) and np.array_equal(gc, cnt), (what, aim)

    firsts = set()
    try:
        for aim in aims:
            # rounds of the whole text: the first one would end at `aim`
            cuts, _ = sh.hc[0].fastq_cuts(buf.data_ptr(), len(data), aim)
            assert cuts[0] == max(e for e in ends if e <= aim)
            firsts.add(cuts[0])
            bounds = [0] + cuts + [len(data)]

            def rounds():
                for a, b in zip(bounds, bounds[1:]):
                    sh.extract(0, aligned_text(buf.data_ptr() + a, b - a, stage), b - a, a == 0, b == len(data), None)
            check(rounds, aim, "round")
        assert firsts == set(ends[19:23])
        # pieces of a share whose first nominal end is `aim`
        with tempfile.TemporaryDirectory() as d:
            path = os.path.join(d, "a.fq")
            with open(path, "wb") as f:
                f.write(data)
            share = split.plan_file(path, 0, 1, k)
            for aim in aims:
                reader = ShareReader(path, share, aim + ShareReader.CR_SLACK, records=True)   # (the slack is 4096 here)
                got = []

                def pieces():
                    try:
                        for i in range(reader.n_pieces):
                            hptr, n, begin, end = reader.read(i)
                            got.append(C.string_at(hptr, n))
                            assert lib.jfgpu_memcpy_h2d(C.c_void_p(stage.data_ptr()), C.c_void_p(hptr), n, None) == 0
                            torch.cuda.synchronize()
                            reader.release(i)
                            sh.extract(0, stage.data_ptr(), n, begin, end, share.fmt)
                    finally:
                        reader.close()
                check(pieces, aim, "piece")
                assert len(got[0]) == max(e for e in ends if e <= aim) and b"".join(got) == data, aim
    finally:
        sh.close()


def test_if_fallback_recounts_both_passes(cuda, workdir, inputs):
    """A FASTQ file whose cut fools the local rule, given to --if and counted under -Q: the newline check fails, the shards
    are cleared and both passes (PRIME over the --if file, UPDATE over the inputs) are counted again with whole files; the
    result is the single-GPU count of the same switches."""
    from test_gpu_split_multi import _fooled_fastq
    from jellyfish_b200 import HashCounter
    world = 4
    fq = os.path.join(workdir, "qmf_fooled.fq")
    with open(fq, "wb") as fh:
        fh.write(_fooled_fastq(world, 21))
    eng = {"k": 21, "canonical": True, "size": 1 << 20, "min_qual": ord("5")}
    ifs, paths = [fq], [fq, inputs["reads_q.fq"]]
    h, b, fell_back = _count(cuda, eng, ifs, paths, world, False, "split")
    assert fell_back
    with HashCounter(1 << 20, 7, k=21, canonical=True, min_qual="5") as one:
        one.set_op(HashCounter.OP_PRIME)
        one.add_files(ifs)
        one.set_op(HashCounter.OP_UPDATE)
        one.add_files(paths)
        one.done()
        assert b == one.dump_records()
