"""The SAM corpus and the BAM model without a GPU: every cell lands where sam_corpus claims, the BAM model (written from the
SAM specification) agrees with the SAM model through sam_to_bam, and hand-written BAM records decode as the specification
says."""
import struct

import pytest

import sam_corpus as sc
import sam_tools
from sam_tools import FormatError
from test_gpu_sam import CORNERS


def _for_bam(sam):
    """the lines sam_to_bam can write: "\\n" line ends, no empty RNAME/POS fields"""
    return b"".join(ln + b"\n" for ln in sam.replace(b"\r\n", b"\n").split(b"\n") if ln and not ln.startswith(b"\t"))


def _upper_seq(fq):
    """BAM keeps no case: the SEQ lines of a FASTQ in upper case"""
    lines = fq.split(b"\n")
    return b"\n".join(ln.upper() if i % 4 == 1 else ln for i, ln in enumerate(lines))


@pytest.mark.parametrize("name", sorted(set(CORNERS) - {"empty", "header_only"}) + ["block"])
def test_bam_model_matches_sam_model(name):
    sam = _for_bam(sc.corpus_block() if name == "block" else CORNERS[name])
    assert sam_tools.sam_model_fastq(sam)
    assert sc.bam_model_fastq(sam_tools.sam_to_bam(sam)) == _upper_seq(sam_tools.sam_model_fastq(sam))


def test_bam_records_decode_as_specified():
    hdr = sc.bam_header(refs=((b"chr1", 100), (b"c" * 300, 5)))
    recs = [
        sc.bam_record(codes=[1, 2, 4], qual=[0, 1, 40]),                                   # odd l_seq: the pad nibble is not read
        sc.bam_record(codes=list(range(16)), qual=[0xFF, 222, 223, 224] + [93] * 12),     # '=' and 3, 5 ... 15 are N; phred wraps
        sc.bam_record(codes=[]),                                                           # l_seq = 0: nothing
        sc.bam_record(codes=[8, 8], name=b"n" * 254, n_cigar=3000, tags=b"XAZ" + b"y" * 5000 + b"\0"),
    ]
    want = (b"@\nACG\n+\n!\"I\n"
            + b"@\nNACNGNNNTNNNNNNN\n+\n" + bytes([0x20, 255, 0, 1]) + b"~" * 12 + b"\n"
            + b"@\nTT\n+\n??\n")
    assert sc.bam_model_fastq(hdr + b"".join(recs)) == want
    offs = [len(hdr) + sum(len(r) for r in recs[:i]) for i in range(len(recs))]
    assert [o for o, _ in sc.bam_model_records(hdr + b"".join(recs))] == [offs[0], offs[1], offs[3]]


def test_bam_model_errors():
    hdr = sc.bam_header()
    good = sc.bam_record(codes=[1, 2])
    cases = [
        (b"BAM\2" + hdr[4:] + good, 0, "Invalid BAM magic"),
        (hdr[:10], 0, "Truncated BAM header"),
        (hdr + good + struct.pack("<I", 31) + b"\0" * 31, len(hdr) + len(good), "below the 32 bytes"),
        (hdr + good + sc.bam_record(codes=[1, 2], l_seq=3), len(hdr) + len(good), "run past its block_size"),
        (hdr + good + sc.bam_record(codes=[1, 2], l_seq=-1), len(hdr) + len(good), "run past its block_size"),
        (hdr + good + good[:-1], len(hdr) + len(good), "Truncated BAM record"),
        (hdr + good + good[:3], len(hdr) + len(good), "Truncated BAM record"),
    ]
    for data, at, what in cases:
        with pytest.raises(FormatError) as ei:
            sc.bam_model_fastq(data)
        assert ei.value.offset == at and what in ei.value.what, (ei.value, at, what)
    # a record whose QUAL ends exactly at block_size is whole
    assert sc.bam_model_fastq(hdr + good) == b"@\nAC\n+\n??\n"


def test_sam_model_error_offsets():
    good = sc.rec(b"r", b"ACGT", b"IIII")
    for data, at, what in [
        (good + b"x\t1\n" + good, len(good), "fewer than 11 fields"),
        (b"@HD\n" + good * 2 + sc.rec(b"r", b"ACGT", b"III"), 4 + 2 * len(good), "different lengths"),
        (good + b"\r\r\n", len(good), "fewer than 11 fields"),
        (good + b"\t" * 9 + b"\n", len(good), "fewer than 11 fields"),
    ]:
        with pytest.raises(FormatError) as ei:
            sam_tools.sam_model_fastq(data)
        assert ei.value.offset == at and what in ei.value.what
    assert sam_tools.sam_model_fastq(good + b"\t" * 10 + b"\n" + b"\r\n\n") == b"@\nACGT\n+\nIIII\n"


def test_caps():
    assert sc.sam_caps(0) == (32 << 20, 32 << 20)
    assert sc.sam_caps(100) == (64, 64)
    assert sc.sam_caps(1000) == (496, 496)
    assert sc.sam_caps(4 << 30) == (1 << 30, 1 << 30)


def test_block_lanes():
    """Across the block's lines, tab 9, tab 10, tab 11, '\\r' and '\\n' each take every lane of the 32-byte stride."""
    block = sc.corpus_block()
    lanes = {k: set() for k in ("t9", "t10", "t11", "cr", "nl")}
    at = 0
    for ln in block.split(b"\n")[:-1]:
        tabs = [i for i, c in enumerate(ln) if c == 9]
        if len(tabs) >= 10 and not ln.startswith(b"@"):
            lanes["t9"].add(tabs[8] % 32)
            lanes["t10"].add(tabs[9] % 32)
            if len(tabs) >= 11:
                lanes["t11"].add(tabs[10] % 32)
            if ln.endswith(b"\r"):
                lanes["cr"].add((len(ln) - 1) % 32)
            lanes["nl"].add(len(ln) % 32)
        at += len(ln) + 1
    for k, v in lanes.items():
        assert v == set(range(32)), (k, sorted(set(range(32)) - v))


def test_pads_reach_every_word_residue_and_tile_edge():
    block = sc.corpus_block()
    cap = sc.sam_caps(0)[1]
    starts = set()
    word_end_lines = set()
    for p in range(48):
        text = sc.padded(p, block, p % 2 == 0)
        walk = sc.host_walk(text, cap)
        assert len(walk) == 1 and walk[0].lo == 0
        for s in sc.line_starts(text):
            starts.add((p, walk[0].rel(s) % sc.WORD))
        word_end_lines |= {i - p for i, c in enumerate(text) if c == 10 and i % 16 == 15 and i >= p}
    assert {r for _, r in starts} == set(range(16))
    assert word_end_lines >= {i for i, c in enumerate(block) if c == 10}      # every newline of the block ends a word
    pads = sc.tile_pads(block)
    for x in [i for i, c in enumerate(block) if c == 10]:
        for d in (-1, 0, 1):
            assert sc.padded(sc.TILE - 1 - x + d, block)[sc.TILE - 1 + d] == 10
            assert sc.TILE - 1 - x + d in pads


@pytest.mark.parametrize("mbb", [600, 1000, 4000])
def test_device_walk_reaches_every_lo(mbb):
    """the device batches of the padded block start at every residue of a 16-byte word, behind a newline in the same word"""
    cap = sc.sam_caps(mbb)[1]
    los = set()
    for p in range(0, 48, 7) if mbb < 4096 else range(48):
        text = sc.padded(p, sc.corpus_block())
        walk = sc.device_walk(text, cap)
        for b in walk[1:]:
            assert text[b.off - 1] == 10
        los |= {b.lo for b in walk}
        assert all(b.used <= cap for b in walk)
    assert los == set(range(16)), sorted(set(range(16)) - los)


def test_fixed_sam_matches_model():
    sam, fq, w = sc.fixed_sam(300, 7, zero_every=5, crlf_every=3, star_qual_every=4, head=45)
    assert sam_tools.sam_model_fastq(sam) == fq
    assert len(sam) == 45 + 300 * w


def test_fixed_fields_read_back():
    """the benchmark-size case's FASTQ, made from the columns of its lines, is the text model's"""
    import numpy as np
    from test_gpu_sam_transcode import MIDS, TAGS
    n, R = 400, 150
    rng = np.random.default_rng(3)
    seq = np.frombuffer(b"ACGT", np.uint8)[rng.integers(0, 4, (n, R))]
    qual = rng.integers(33, 75, (n, R), dtype=np.uint8)
    zero, crlf, sq = sc.kinds(n, crlf_every=13, star_qual_every=97)
    lines = sc.fixed_lines(np, seq, qual, 380, zero, crlf, sq, mids=MIDS, tail=TAGS)
    s2, q2 = sc.fixed_fields(np, lines, R, crlf, sq, TAGS)
    fq = sc.fixed_fastq(np, s2, q2, zero, sq)
    assert (s2 == seq).all() and fq.tobytes() == sam_tools.sam_model_fastq(lines.tobytes())


def test_short_lines_stay_under_rec_cap():
    """A batch of 11-byte and 13-byte lines never has more line starts than the transcode's rec_cap (in_cap / 11 + 2), and
    lines under 11 bytes that overflow it start behind the first short line"""
    for mbb in (1 << 12, 1 << 16):
        in_cap, cap = sc.sam_caps(mbb)
        text = (b"\t" * 10 + b"\n" + b"\t" * 9 + b"A\tI\n") * (cap // 12)
        for walk in (sc.host_walk(text, cap), sc.device_walk(text, cap)):
            for b in walk:
                n = sum(1 for s in sc.line_starts(text[b.off:b.off + b.n]))
                assert n <= in_cap // 11 + 2
