"""The SAM and BAM transcode (jf_sam.cu) byte for byte against the models of sam_tools and sam_corpus.

`HashCounter.sam_stage` returns the FASTQ the transcode writes; every case compares it with the model's records and, on a
mismatch, names the first differing byte, its record, and where that record's line sits in its batch (A, word, tile).
"""
import hashlib
import re
import struct

import pytest

import sam_corpus as sc
import sam_tools
from sam_tools import FormatError

pytestmark = pytest.mark.gpu

SENTINEL = 0xEE
_ENGINES = {}


def _engine(mbb):
    from jellyfish_b200 import HashCounter
    if mbb not in _ENGINES:
        _ENGINES[mbb] = HashCounter(1 << 16, 7, k=21, canonical=True, max_batch_bytes=mbb)
    return _ENGINES[mbb]


@pytest.fixture(scope="module", autouse=True)
def _close_engines():
    yield
    for hc in _ENGINES.values():
        hc.close()
    _ENGINES.clear()


def _dev(data):
    import torch
    return torch.frombuffer(bytearray(data) or bytearray(1), dtype=torch.uint8).cuda()


def stage(hc, data, cuts=(), device=False, bam=False, out_cap=None):
    """The FASTQ of `data` staged in pieces cut at `cuts`, from host or (16-byte aligned) device memory -> (bytes, the
    output buffer: bytes behind the FASTQ still hold SENTINEL)"""
    import torch
    out = torch.full((max(2 * len(data) + 64, 64),), SENTINEL, dtype=torch.uint8, device="cuda")
    cap = out.numel() if out_cap is None else out_cap
    bounds = [0] + list(cuts) + [len(data)]
    total = 0
    for i in range(len(bounds) - 1):
        piece = data[bounds[i]:bounds[i + 1]]
        keep = None
        if device:
            keep = _dev(piece)
            src = ("device", keep.data_ptr(), len(piece))
        else:
            src = piece
        total += hc.sam_stage(src, out.data_ptr() + total, cap - total, begin=i == 0, end=i == len(bounds) - 2, bam=bam)
        torch.cuda.synchronize()
        del keep
    return out[:total].cpu().numpy().tobytes(), out


def check_sam(hc, mbb, text, cuts=(), device=False):
    records = sam_tools.sam_model_records(text)
    got, _ = stage(hc, text, cuts, device)
    cap = sc.sam_caps(mbb)[1]
    walk = sc.device_walk(text, cap) if device else sc.host_walk(text, cap)
    msg = sc.first_mismatch(got, records, walk)
    assert msg is None, "%s cuts %s: %s" % ("device" if device else "host", list(cuts), msg)
    return walk


# ---- the aimed corpus ----------------------------------------------------------------------------------------------------
BLOCK = sc.corpus_block()


@pytest.mark.parametrize("device", [False, True])
@pytest.mark.parametrize("mbb", [0, 600, 1000, 4000, 40000])
def test_corpus_word_residues(mbb, device):
    """Header padding 0 ... 47 puts every line start and newline of the block at every residue of a 16-byte word (every
    second text ends without a newline); small batches start device batches at every residue lo."""
    hc = _engine(mbb)
    los = set()
    for p in range(48):
        walk = check_sam(hc, mbb, sc.padded(p, BLOCK, p % 2 == 0), device=device)
        los |= {b.lo for b in walk}
    if device and 0 < mbb <= 4000:
        assert los == set(range(16)), sorted(los)


@pytest.mark.parametrize("device", [False, True])
@pytest.mark.parametrize("mbb", [0, 40000])
def test_corpus_tile_edges(mbb, device):
    """Every newline of the block at the last byte of a 16 KB tile, one byte before it and one after."""
    hc = _engine(mbb)
    cap = sc.sam_caps(mbb)[1]
    hit = 0
    for p in sc.tile_pads(BLOCK, every=1 if mbb == 0 else 3):
        text = sc.padded(p, BLOCK)
        walk = check_sam(hc, mbb, text, device=device)
        if len(text) > sc.TILE:
            i, b = sc.batch_of(walk, sc.TILE - 1)
            hit += text[sc.TILE - 1] == 10 and b.rel(sc.TILE - 1) == sc.TILE - 1
    assert hit >= 1 and cap > sc.TILE


@pytest.mark.parametrize("device", [False, True])
def test_corpus_cut_across_calls(device):
    """One text cut into two calls at every byte of a window at its start and around a tile edge, and into many calls."""
    hc = _engine(40000 if device else 4000)
    mbb = 40000 if device else 4000
    text = sc.padded(sc.TILE - 40, BLOCK, False)
    for c in list(range(0, 240)) + list(range(sc.TILE - 60, sc.TILE + 200)):
        check_sam(hc, mbb, text, cuts=[c], device=device)
    check_sam(hc, mbb, text, cuts=list(range(7, len(text), 311)), device=device)
    check_sam(hc, mbb, text, cuts=list(range(1, 300)), device=device)


# ---- record and tile counts ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [1, 1023, 1024, 1025, 262143, 262144, 262145, 300001])
def test_record_counts(n):
    """n one-base lines in one batch, every third with SEQ '*' and QUAL '*' (zero-length records)"""
    hc = _engine(0)
    sam, fq, _ = sc.fixed_sam(n, 1, zero_every=3, head=5, seed=n)
    walk = sc.host_walk(sam, sc.sam_caps(0)[1])
    assert len(walk) == 1
    for device in (False, True):
        got, _ = stage(hc, sam, device=device)
        assert got == fq, (device, _diff(got, fq, 2 * 1 + 6))


def _diff(got, want, rec):
    i = next((j for j in range(min(len(got), len(want))) if got[j] != want[j]), min(len(got), len(want)))
    return "sizes %d / %d, first difference at byte %d (record %d)" % (len(got), len(want), i, i // rec)


@pytest.mark.parametrize("tiles", [1024, 2048])
@pytest.mark.parametrize("d", [-1, 0, 1])
def test_tile_counts(tiles, d):
    """One batch of tiles * 16 KB + d bytes: the tile scan just under, at and just over 1024 and 2048 tiles"""
    size = tiles * sc.TILE + d
    mbb = 256 << 20
    hc = _engine(mbb)
    w = 9 + 2 * 50 + 3
    n = (size - 64) // w
    sam, fq, w2 = sc.fixed_sam(n, 50, zero_every=7, star_qual_every=5, head=size - n * w, seed=tiles + d)
    assert w2 == w and len(sam) == size
    walk = sc.host_walk(sam, sc.sam_caps(mbb)[1])
    assert len(walk) == 1 and walk[0].tiles == tiles + (d > 0)
    for device in (False, True):
        got, _ = stage(hc, sam, device=device)
        assert got == fq, (device, _diff(got, fq, 2 * 50 + 6))


@pytest.mark.parametrize("device", [False, True])
@pytest.mark.parametrize("mbb", [1 << 12, 1 << 16])
def test_shortest_lines_fill_batches(mbb, device):
    """Batches of nothing but 11-byte lines (10 tabs) and 13-byte one-base lines pass; one 10-byte line among them fails at
    its offset."""
    hc = _engine(mbb)
    cap = sc.sam_caps(mbb)[1]
    text = (b"\t" * 10 + b"\n" + b"\t" * 9 + b"A\tI\n") * (3 * cap // 24) + b"\t" * 10 + b"\n"
    check_sam(hc, mbb, text, device=device)
    at = len(text) // 2 // 24 * 24 + 11
    bad = text[:at] + b"\t" * 9 + b"\n" + text[at:]
    _check_error(hc, bad, at, device=device)


# ---- errors --------------------------------------------------------------------------------------------------------------
def _check_error(hc, data, at=None, device=False, bam=False, what=None):
    """The stage fails with JFGPU_ERR_FORMAT, names byte `at` (default: the model's offset), and writes nothing past the
    records of the batches in front of the failing one"""
    from jellyfish_b200 import JellyfishError, _lib as L
    model = sc.bam_model_records if bam else sam_tools.sam_model_records
    with pytest.raises(FormatError) as me:
        model(data)
    at = me.value.offset if at is None else at
    assert at == me.value.offset
    import torch
    out = torch.full((2 * len(data) + 64,), SENTINEL, dtype=torch.uint8, device="cuda")
    keep = _dev(data) if device else None
    with pytest.raises(JellyfishError) as ei:
        hc.sam_stage(("device", keep.data_ptr(), len(data)) if device else data, out.data_ptr(), out.numel(), bam=bam)
    torch.cuda.synchronize()
    msg = str(ei.value)
    assert ei.value.code == L.ERR_FORMAT, msg
    assert re.search(r"at byte %d of the " % at, msg), (msg, at)
    if what:
        assert what in msg, msg
    written = out.cpu().numpy().tobytes().rstrip(bytes([SENTINEL]))
    good = b"".join(r for o, r in model(data[:at]))
    assert good.startswith(written), "output written past the records in front of the bad one"
    assert written == b"" or written.endswith(b"\n")


def _sam_lines(n, seed):
    return [sc.rec(b"r%d" % i, sc._bases(20 + i % 9, i + seed), sc._qual(20 + i % 9, i)) for i in range(n)]


SAM_BAD = {
    "few_fields": b"r\t0\tchr1\t1\t60\t4M\t*\t0\tACGT\tIIII\n",
    "qual_len": sc.rec(b"r", b"ACGT", b"III"),
    "nine_tabs": b"\t" * 9 + b"\n",
    "cr_only": b"\r\r\n",
    "short_lines": b"x\n" * 2000,             # more line starts than the batch's record capacity
}


@pytest.mark.parametrize("device", [False, True])
@pytest.mark.parametrize("where", [2, 9, 61])
@pytest.mark.parametrize("bad", sorted(SAM_BAD))
def test_sam_error_offsets(bad, where, device):
    """A bad line in the first, second or a later batch (about 8 lines per batch): the message names its offset."""
    hc = _engine(1000)
    lines = _sam_lines(90, where)
    text = b"@HD\tVN:1.6\n" + b"".join(lines[:where]) + SAM_BAD[bad] + b"".join(lines[where:])
    _check_error(hc, text, device=device)
    # the engine continues with the next file
    check_sam(hc, 1000, b"".join(lines), device=device)


def _bam_records(n, seed):
    return [sc.bam_record(codes=[(1, 2, 4, 8)[(i * j + seed) % 4] for j in range(11 + i % 9)], name=b"r%d" % i) for i in range(n)]


BAM_BAD = {
    "l_seq_past_block": lambda: sc.bam_record(codes=[1, 2, 4], l_seq=4),
    "l_seq_negative": lambda: sc.bam_record(codes=[1, 2, 4], l_seq=-3),
    "names_past_block": lambda: sc.bam_record(codes=[1, 2], name=b"n" * 40, block_size=50),
    "block_size_31": lambda: struct.pack("<I", 31) + b"\0" * 31,
    "truncated": None,
}


@pytest.mark.parametrize("where", [1, 12, 45])
@pytest.mark.parametrize("bad", sorted(BAM_BAD))
def test_bam_error_offsets(bad, where):
    hc = _engine(1000)
    recs = _bam_records(60, where)
    hdr = sc.bam_header()
    if bad == "truncated":
        data = hdr + b"".join(recs[:where]) + recs[where][:-3]
    else:
        data = hdr + b"".join(recs[:where]) + BAM_BAD[bad]() + b"".join(recs[where:])
    _check_error(hc, data, bam=True)
    got, _ = stage(hc, hdr + b"".join(recs), bam=True)
    assert got == sc.bam_model_fastq(hdr + b"".join(recs))


# ---- BAM corners ---------------------------------------------------------------------------------------------------------
def _bam_corners():
    recs = [
        sc.bam_record(codes=[1, 2, 4], qual=[0, 1, 40]),                                 # odd l_seq
        sc.bam_record(codes=list(range(16)) * 3, qual=[0xFF, 222, 223, 224, 0, 93] * 8),  # '=', 3, 5 ... 15; phred wraps
        sc.bam_record(codes=[]),                                                         # l_seq = 0
        sc.bam_record(codes=[8, 1] * 20, name=b"n" * 254),                               # a 255-byte read name
        sc.bam_record(codes=[4] * 33, n_cigar=3000),                                     # thousands of CIGAR ops
        sc.bam_record(codes=[2] * 9, tags=b"XAZ" + b"t" * 20000 + b"\0"),                # long tags
        sc.bam_record(codes=[1, 8, 8, 1, 2]),                                            # QUAL ends at block_size
    ]
    return sc.bam_header(refs=((b"chr1", 1000), (b"c" * 300, 5))), recs


def test_bam_corners_cut_everywhere():
    """The corners whole, and cut across two calls at every byte of the header and of a record's block_size field, and at
    every byte of the first records (the host tail path)"""
    hc = _engine(0)
    hdr, recs = _bam_corners()
    data = hdr + b"".join(recs)
    want = sc.bam_model_fastq(data)
    assert stage(hc, data, bam=True)[0] == want
    r4 = len(hdr) + sum(len(r) for r in recs[:4])
    for c in list(range(1, len(hdr) + 200)) + list(range(r4 - 2, r4 + 7)):
        got = stage(hc, data, cuts=[c], bam=True)[0]
        assert got == want, "cut at %d: %s" % (c, sc.first_mismatch(got, sc.bam_model_records(data)))
    assert stage(hc, data, cuts=range(1, len(data), 97), bam=True)[0] == want


def test_bam_record_of_exactly_cap_bytes():
    """A record of exactly `cap` bytes is one batch; one of cap + 1 bytes is refused"""
    from jellyfish_b200 import JellyfishError, _lib as L
    mbb = 1000
    hc = _engine(mbb)
    cap = sc.sam_caps(mbb)[1]
    hdr = sc.bam_header()
    small = sc.bam_record(codes=[1, 2])
    base = len(sc.bam_record(codes=[1] * 100))
    fit = sc.bam_record(codes=[1] * 100, tags=b"x" * (cap - base))
    assert len(fit) == cap
    for data in (hdr + small + fit + small, hdr + fit):
        for cuts in ([], [len(hdr) + 2], [len(data) - 1]):
            assert stage(hc, data, cuts=cuts, bam=True)[0] == sc.bam_model_fastq(data)
    over = sc.bam_record(codes=[1] * 100, tags=b"x" * (cap + 1 - base))
    with pytest.raises(JellyfishError) as ei:
        stage(hc, hdr + small + over, bam=True)
    assert ei.value.code == L.ERR_FORMAT and "longer than the staging buffer" in str(ei.value)


def test_bam_header_errors():
    from jellyfish_b200 import JellyfishError, _lib as L
    hc = _engine(0)
    hdr = sc.bam_header()
    rec = sc.bam_record(codes=[1, 2])
    for data, what in ((b"BAM\2" + hdr[4:] + rec, "Invalid BAM magic"), (hdr[:-3], "Truncated BAM header"),
                       (hdr[:9], "Truncated BAM header")):
        with pytest.raises(FormatError):
            sc.bam_model_fastq(data)
        with pytest.raises(JellyfishError) as ei:
            stage(hc, data, bam=True)
        assert ei.value.code == L.ERR_FORMAT and what in str(ei.value)


# ---- the jfgpu_sam_stage contract ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("bam", [False, True])
def test_out_cap(bam):
    from jellyfish_b200 import JellyfishError, _lib as L
    hc = _engine(1000)
    text = b"".join(_sam_lines(40, 3))
    data = sam_tools.sam_to_bam(text) if bam else text
    want = sam_tools.sam_model_fastq(text)
    got, _ = stage(hc, data, bam=bam, out_cap=len(want))
    assert got == want
    with pytest.raises(JellyfishError) as ei:
        stage(hc, data, bam=bam, out_cap=len(want) - 1)
    assert ei.value.code == L.ERR_ARG
    assert stage(hc, data, bam=bam)[0] == want                  # and the next file starts clean


def test_count_between_stage_calls():
    """A SAM file counted with add_sam_text between two stage calls of another leaves both unchanged."""
    import torch
    from jellyfish_b200 import HashCounter
    text = sc.padded(5, BLOCK)
    other = b"".join(_sam_lines(70, 9))
    want = sam_tools.sam_model_fastq(text)
    with HashCounter(1 << 16, 7, k=17, canonical=True, max_batch_bytes=1000) as hc:
        out = torch.full((2 * len(text),), SENTINEL, dtype=torch.uint8, device="cuda")
        c = len(text) // 2 + 3
        n1 = hc.sam_stage(text[:c], out.data_ptr(), out.numel(), begin=True, end=False)
        hc.add_sam_text(other)
        n2 = hc.sam_stage(text[c:], out.data_ptr() + n1, out.numel() - n1, begin=False, end=True)
        torch.cuda.synchronize()
        assert out[:n1 + n2].cpu().numpy().tobytes() == want
        hc.done()
        counted = hc.dump_records()
    with HashCounter(1 << 16, 7, k=17, canonical=True, max_batch_bytes=1000) as hc:
        hc.add_text(sam_tools.sam_model_fastq(other))
        hc.done()
        assert hc.dump_records() == counted


@pytest.mark.parametrize("device", [False, True])
def test_begin_after_failed_file(device):
    hc = _engine(1000)
    lines = _sam_lines(40, 1)
    bad = b"".join(lines[:20]) + SAM_BAD["few_fields"] + b"".join(lines[20:])
    _check_error(hc, bad, device=device)
    # the failed file's carry is gone: a file cut inside a line follows
    text = b"".join(lines)
    check_sam(hc, 1000, text, cuts=[len(lines[0]) + 5], device=device)


# ---- benchmark size ------------------------------------------------------------------------------------------------------
READ = 150
MIDS = (b"\t0\tchr1\t1234567\t60\t150M\t*\t0\t0\t", b"\t4\t*\t0\t0\t*\t*\t0\t0\t", b"\t16\tchr1\t1234567\t60\t150M\t*\t0\t0\t",
        b"\t256\tchr1\t1234567\t60\t150M\t*\t0\t0\t")
TAGS = b"\tNM:i:1\tMD:Z:75A74\tAS:i:145\tRG:Z:grp1"


def test_benchmark_size():
    """scripts/sam_bench.py's shape: 5 M reads of 150 bases (FLAG 0/4/16/256, every 97th QUAL '*', every 13th line CRLF),
    about 1.9 GB in HBM, staged at the default batch and at max_batch_bytes = 2 GB (in_cap = 1 GB: about 65 000 tiles and
    2.8 M records per batch); then counted at k = 21 -C, equal to the count of its FASTQ."""
    import torch
    from jellyfish_b200 import HashCounter
    for hc in _ENGINES.values():            # (an engine of 2 GB batches holds about 71 GB of HBM)
        hc.close()
    _ENGINES.clear()
    n, width = 5_000_000, 380
    g = torch.Generator(device="cuda").manual_seed(5)
    seq = torch.tensor(list(b"ACGT"), dtype=torch.uint8, device="cuda")[torch.randint(0, 4, (n, READ), device="cuda", generator=g)]
    qual = torch.randint(33, 75, (n, READ), device="cuda", generator=g, dtype=torch.uint8)
    zero, crlf, sq = (torch.from_numpy(m).cuda() for m in sc.kinds(n, crlf_every=13, star_qual_every=97))
    lines = sc.fixed_lines(torch, seq, qual, width, zero, crlf, sq, mids=MIDS, tail=TAGS)
    del seq, qual
    head = b"@HD\tVN:1.6\tSO:unsorted\n@SQ\tSN:chr1\tLN:248956422\n"
    sam = torch.empty(len(head) + lines.numel(), dtype=torch.uint8, device="cuda")
    sam[:len(head)] = torch.frombuffer(bytearray(head), dtype=torch.uint8).cuda()
    sam[len(head):] = lines.reshape(-1)
    del lines
    torch.cuda.empty_cache()
    body = sam[len(head):].view(n, width)

    def expected(a, b):
        """the FASTQ of lines [a, b), from the columns fixed_lines wrote them to (test_sam_corpus_cpu pins it to the model)"""
        s, q = sc.fixed_fields(torch, body[a:b], READ, crlf[a:b], sq[a:b], TAGS)
        return sc.fixed_fastq(torch, s, q, zero[a:b], sq[a:b])
    assert sam_tools.sam_model_fastq(body[:300].cpu().numpy().tobytes()) == expected(0, 300).cpu().numpy().tobytes()
    rec = 2 * READ + 6
    out = torch.empty(n * rec, dtype=torch.uint8, device="cuda")
    for mbb in (2 << 30, 0):
        in_cap, cap = sc.sam_caps(mbb)
        if mbb:
            assert cap == 1 << 30 and -(-cap // sc.TILE) == 65536 and (cap - len(head)) // width + 1 > 2_800_000
        out.fill_(SENTINEL)
        with HashCounter(1 << 16, 7, k=21, canonical=True, max_batch_bytes=mbb) as hc:
            got = hc.sam_stage(("device", sam.data_ptr(), sam.numel()), out.data_ptr(), out.numel())
        torch.cuda.synchronize()
        assert got == out.numel()
        for a in range(0, n, 1 << 20):
            b = min(n, a + (1 << 20))
            o, want = out.view(n, rec)[a:b], expected(a, b)
            bad = (o != want).any(dim=1).nonzero()
            if bad.numel():
                r = int(bad[0])
                col = int((o[r] != want[r]).nonzero()[0])
                r += a
                pos = len(head) + r * width          # (no zero-length lines here: record r is line r)
                raise AssertionError("mbb %d: first difference at output byte %d (record %d, byte %d), the line at file byte %d; "
                                     "%s: got %r want %r" % (mbb, r * rec + col, r, col, pos,
                                                             _fixed_where(sam.numel(), len(head), width, cap, pos),
                                                             bytes(o[r - a].cpu().tolist())[:40], bytes(want[r - a].cpu().tolist())[:40]))
        torch.cuda.empty_cache()
    del out
    fq = torch.cat([expected(a, min(n, a + (1 << 20))).reshape(-1) for a in range(0, n, 1 << 20)])
    torch.cuda.empty_cache()

    def count(dev, is_sam):
        h = hashlib.md5()
        with HashCounter(1 << 30, 7, k=21, canonical=True) as hc:
            hc.add_device_text(dev.data_ptr(), dev.numel(), sam=is_sam)
            st = hc.done()
            torch.cuda.synchronize()
            hc.dump_records(sink=h.update)
        return st, h.hexdigest()
    s1, h1 = count(sam, True)
    del sam
    s2, h2 = count(fq, False)
    keys = ("kmers", "inserted", "distinct", "overflowed")
    assert {k: s1[k] for k in keys} == {k: s2[k] for k in keys} and h1 == h2
    assert s1["kmers"] == n * (READ - 21 + 1)


def _fixed_where(size, head, width, cap, pos):
    """sc.where for device text of `head` bytes of header and then lines of `width` bytes, without reading it"""
    walk, off = [], 0
    while off < size:
        ln = min(cap, size - off)
        used = ln if off + ln == size else head + (off + ln - head) // width * width - off
        walk.append(sc.Batch(off, off & 15, ln, used))
        off += used
    return sc.where(walk, pos)
