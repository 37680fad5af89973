"""The SAM / BAM split plan (jellyfish_b200/split_sam.py) against a model that walks the whole file: BAM cuts are the first
record at or after the first BGZF block at or after each nominal cut, SAM cuts are line starts, the shares' pieces put
together are the file, a record chain imitated inside a tag fools the local rule, and broken blocks
are errors.  CPU only."""
import random
import struct

import pytest

import sam_tools
from jellyfish_b200 import split_sam


def _fastq(n, seed, lo=20, hi=300):
    rng = random.Random(seed)
    out = []
    for i in range(n):
        ln = rng.randint(lo, hi)
        out.append(b"@r%d\n%s\n+\n%s\n" % (i, bytes(rng.choice(b"ACGTN") for _ in range(ln)), bytes(rng.randint(35, 74) for _ in range(ln))))
    return b"".join(out)


def _bgzf_at(data, cuts):
    """BGZF of data cut at the given inflated offsets, then the end-of-file block -> (file, [(block offset, inflated start)])."""
    out, blocks, pos = b"", [], 0
    for c in list(cuts) + [len(data)]:
        if c > pos:
            blocks.append((len(out), pos))
            out += sam_tools.bgzf_block(data[pos:c])
            pos = c
    return out + sam_tools.BGZF_EOF, blocks


def _chain(stream):
    """The inflated offsets of every record (the model: the header, then the block_size chain)."""
    o = 8 + struct.unpack_from("<i", stream, 4)[0]
    n_ref = struct.unpack_from("<i", stream, o)[0]
    o += 4
    for _ in range(n_ref):
        o += 8 + struct.unpack_from("<i", stream, o)[0]
    recs = []
    while o < len(stream):
        recs.append(o)
        o += 4 + struct.unpack_from("<I", stream, o)[0]
    assert o == len(stream)
    return recs


def _model_start(blocks, size, stream, recs, a):
    if a <= 0:
        return (0, 0)
    starts = [b for b, _ in blocks]
    c = next((b for b in starts if b >= a), None)
    if c is None:
        return (size, 0)
    u = dict(blocks)[c]
    r = next((x for x in recs if x >= u), None)
    if r is None:
        return (size, 0)
    b, s = max((bs for bs in blocks if bs[1] <= r), key=lambda bs: bs[1])
    return (b, r - s)


def _bam(seed, block, n=400):
    stream = sam_tools.sam_to_bam(sam_tools.fastq_to_sam(_fastq(n, seed)))
    rng = random.Random(seed)
    cuts, p = [], 0
    while True:
        p += rng.randint(block // 2, block)
        if p >= len(stream):
            break
        cuts.append(p)
    data, blocks = _bgzf_at(stream, cuts)
    return data, blocks, stream


@pytest.mark.parametrize("seed,block", [(1, 3000), (2, 700), (3, 20000), (4, 150)])
def test_bam_cuts_match_the_chain_model(seed, block):
    data, blocks, stream = _bam(seed, block)
    recs = _chain(stream)
    rd = lambda off, n: data[off:off + n]
    n_ref, hlen = split_sam.bam_header(rd, len(data))
    assert n_ref == 2 and hlen == recs[0]
    header_end = split_sam._Inflated(rd, len(data), 0).position(hlen)
    for a in sorted((set(range(1, len(data), 97)) | {b for b, _ in blocks} | {b + 1 for b, _ in blocks}) - {0}):
        got = split_sam.bam_share_start(rd, len(data), n_ref, header_end, a)
        assert got == max(_model_start(blocks, len(data), stream, recs, a), header_end), a
    for world in range(2, 9):
        shares = [split_sam.plan_bam_share(rd, len(data), r, world) for r in range(world)]
        assert shares[0].start == (0, 0) and shares[-1].end == (len(data), 0)
        for r in range(world - 1):
            assert shares[r].end == shares[r + 1].start


@pytest.mark.parametrize("world", [2, 3, 5, 8])
def test_bam_share_pieces_put_together_are_the_stream(tmp_path, world):
    data, blocks, stream = _bam(7, 2500)
    path = str(tmp_path / "x.bam")
    open(path, "wb").write(data)
    got = b""
    for r in range(world):
        kind, share = split_sam.plan_file(path, r, world)
        assert kind == "bam"
        rd = split_sam.BamShareReader(path, share, 5000, threads=3)
        parts = []
        for i in range(rd.n_pieces):
            rd.prefetch(i)
            b, begin, end = rd.read(i)
            assert begin == (i == 0) and end == (i == rd.n_pieces - 1)
            assert len(b) <= 5000 + 65536 + len(split_sam.EMPTY_BAM_HEADER)
            parts.append(b)
        rd.close()
        piece = b"".join(parts)
        if r and piece:
            assert piece.startswith(split_sam.EMPTY_BAM_HEADER)
            piece = piece[len(split_sam.EMPTY_BAM_HEADER):]
        got += piece
    assert got == stream


def test_sam_text_cuts_are_line_starts():
    sam = sam_tools.fastq_to_sam(_fastq(300, 9))
    rd = lambda off, n: sam[off:off + n]
    for world in range(2, 9):
        cuts = [split_sam.plan_sam_share(rd, len(sam), r, world) for r in range(world)]
        assert cuts[0][0] == 0 and cuts[-1][1] == len(sam)
        for (s, e), (s2, _) in zip(cuts, cuts[1:]):
            assert e == s2
            assert s == 0 or sam[s - 1:s] == b"\n"
        assert b"".join(sam[s:e] for s, e in cuts) == sam


def _fake_records(n):
    """n records that parse consistently: refID 0, one-byte name, four bases."""
    body = struct.pack("<iiBBHHHiiii", 0, 5, 2, 60, 4680, 0, 0, 4, -1, -1, 0) + b"f\0" + b"\x12\x48" + b"\x1e" * 4
    return (struct.pack("<I", len(body)) + body) * n


def imitation_bam():
    """A BAM file whose second block starts inside a record, right where that record's B:C tag holds a chain of fake records
    that ends with the record: the local rule takes the fake chain for a cut.  -> (file bytes, inflated offset of the fake
    chain)."""
    base = sam_tools.sam_to_bam(sam_tools.fastq_to_sam(_fastq(100, 11, 100, 200)))
    recs = _chain(base)
    host_at = recs[-20]
    fake = _fake_records(40)
    tag = b"XBBC" + struct.pack("<i", len(fake)) + fake
    ln = struct.unpack_from("<I", base, host_at)[0]
    host = struct.pack("<I", ln + len(tag)) + base[host_at + 4:host_at + 4 + ln] + tag
    stream = base[:host_at] + host + base[host_at + 4 + ln:]
    fake_at = host_at + len(host) - len(fake)
    assert fake_at <= 65280                  # (a BGZF block holds at most 64 KB)
    data, _ = _bgzf_at(stream, [fake_at])
    return data, fake_at, stream


def test_imitated_chain_fools_the_cut():
    """(That the check after the count catches it, and the fall-back counts exactly, is tests/test_gpu_split_sam.py.)"""
    data, fake_at, stream = imitation_bam()
    rd = lambda off, n: data[off:off + n]
    # the first block holds most of the (poorly compressible) file: the nominal cut of rank 1 lands in it
    shares = [split_sam.plan_bam_share(rd, len(data), r, 2) for r in range(2)]
    second_block = len(sam_tools.bgzf_block(stream[:fake_at]))
    assert shares[1].start == (second_block, 0)
    # the fake chain is not the file's: rank 0's chain runs past rank 1's start instead of ending there
    recs = _chain(stream)
    assert fake_at not in recs
    assert any(r < fake_at < r + 4 + struct.unpack_from("<I", stream, r)[0] for r in recs)


def test_broken_blocks_are_errors(tmp_path):
    data, blocks, stream = _bam(5, 3000)
    path = str(tmp_path / "t.bam")
    # cut short: the block chain breaks
    open(path, "wb").write(data[:len(data) - 40])
    with pytest.raises(ValueError):
        for r in range(2):
            split_sam.BamShareReader(path, split_sam.plan_file(path, r, 2)[1], 4000).close()
    # a corrupt deflate stream / CRC32
    bad = bytearray(data)
    b, _ = blocks[len(blocks) // 2]
    bad[b + 30] ^= 0xFF
    open(path, "wb").write(bytes(bad))
    with pytest.raises(ValueError):
        for r in range(2):
            rd = split_sam.BamShareReader(path, split_sam.plan_file(path, r, 2)[1], 4000)
            try:
                for i in range(rd.n_pieces):
                    rd.read(i)
            finally:
                rd.close()
    crc = bytearray(data)
    p, _ = blocks[1]
    bs = split_sam.block_size(bytes(crc[p:p + 18]))
    crc[p + bs - 8] ^= 1
    with pytest.raises(ValueError):
        split_sam.inflate_block(bytes(crc[p:p + bs]), p)


def test_kinds(tmp_path):
    import gzip
    sam = sam_tools.fastq_to_sam(_fastq(20, 1))
    files = {"a.sam": sam, "a.sam.gz": gzip.compress(sam), "a.bgzf.sam": sam_tools.bgzf(sam),
             "a.bam": sam_tools.bgzf(sam_tools.sam_to_bam(sam)), "a.cram": b"CRAM\3\0" + b"\0" * 30, "empty": b""}
    want = {"a.sam": "sam", "a.sam.gz": "gz", "a.bgzf.sam": "gz", "a.bam": "bam", "a.cram": "cram", "empty": None}
    for name, body in files.items():
        p = tmp_path / name
        p.write_bytes(body)
        assert split_sam.kind(str(p)) == want[name], name


def test_whole_file_readers(tmp_path):
    """A whole BGZF file (BAM, bgzip'd SAM) is read block by block, anything else whole; the pieces put together are the
    inflated file, and a rank that does not own the file gets no pieces."""
    import gzip
    sam = sam_tools.fastq_to_sam(_fastq(300, 4))
    bam = sam_tools.sam_to_bam(sam)
    files = {"a.bam": (sam_tools.bgzf(bam, block=900), bam, True), "a.bgzf.sam": (sam_tools.bgzf(sam, block=700), sam, True),
             "a.sam.gz": (gzip.compress(sam[:5000]) + gzip.compress(sam[5000:]), sam, False), "a.sam": (sam, sam, False)}
    for name, (body, want, blockwise) in files.items():
        p = str(tmp_path / name)
        open(p, "wb").write(body)
        rd = split_sam.whole_reader(p, True, 3000)
        assert isinstance(rd, split_sam.BamShareReader) == blockwise, name
        assert rd.bam == (name == "a.bam")
        got = b"".join(rd.read(i)[0] for i in range(rd.n_pieces))
        rd.close()
        assert got == want, name
        assert split_sam.whole_reader(p, False, 3000).n_pieces == 0
