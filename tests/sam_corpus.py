"""SAM and BAM inputs aimed at the seams of the transcode (jellyfish_b200/csrc/jf_sam.cu), and models of what it must do.

The transcode reads a batch [lo, hi) from the 16-byte aligned address A at or below its first byte, in 16-byte words and
16 KB tiles, and finds the tabs and line end of every line with ballots over 32-byte strides from the line's start.  Header
lines add nothing to the output, so padding them moves every later byte to each word residue and each side of a tile edge;
QNAME lengths 1 ... 32 move every tab, '\\r' and '\\n' of a line through every lane of the stride.

* bam_model_fastq:   the FASTQ of an inflated BAM stream, from the SAM specification (4.2), independent of sam_to_bam.
* bam_record / bam_header: BAM written from raw fields (any codes, quality bytes, name, CIGAR and tag lengths).
* sam_caps, host_walk, device_walk: the batches the engine cuts a file into (jf_engine.cu, sam_feed_host / sam_feed_device),
  with every line's position relative to its batch's A, word and tile.
* corpus_block, padded, tile_pads: the aimed SAM cells.
* fixed_sam: large SAM of fixed-width lines, with its FASTQ, built with numpy.
"""
import struct

import numpy as np

from sam_tools import FormatError

TILE = 16384
WORD = 16


# ---- BAM -----------------------------------------------------------------------------------------------------------------
def bam_header(text=b"@HD\tVN:1.6\n", refs=((b"chr1", 1000000),)):
    out = b"BAM\1" + struct.pack("<i", len(text)) + text + struct.pack("<i", len(refs))
    for name, ln in refs:
        out += struct.pack("<i", len(name) + 1) + name + b"\0" + struct.pack("<i", ln)
    return out


def bam_record(codes=(), qual=None, name=b"r", n_cigar=1, tags=b"", flag=0, pad_nibble=0xF, l_seq=None, block_size=None):
    """One record from raw fields: 4-bit codes (two per byte; an odd count leaves `pad_nibble` in the low half of the last
    byte), quality bytes (default phred 30), a read name of any length up to 254, n_cigar ops of 1M, raw tag bytes.  l_seq
    and block_size override the true values."""
    codes = list(codes)
    qual = bytes([30] * len(codes)) if qual is None else bytes(qual)
    padded = codes + [pad_nibble] if len(codes) % 2 else codes
    packed = bytes(padded[i] << 4 | padded[i + 1] for i in range(0, len(padded), 2))
    nm = name + b"\0"
    body = struct.pack("<iiBBHHHiiii", 0, 0, len(nm), 60, 4680, n_cigar, flag, len(codes) if l_seq is None else l_seq, -1, -1, 0)
    body += nm + struct.pack("<I", 1 << 4) * n_cigar + packed + qual + tags
    return struct.pack("<I", len(body) if block_size is None else block_size) + body


def _le32(b, at):
    return struct.unpack_from("<I", b, at)[0]


def bam_model_records(stream, cap=None):
    """[(byte offset of the record, its FASTQ record)] of an inflated BAM stream (SAM specification 4.2): the header (magic,
    l_text and text, n_ref, every reference's l_name, name and l_ref), then the block_size chain.  Codes 1/2/4/8 are ACGT,
    any other code N; quality bytes are written as (phred + 33) & 0xff; a record with l_seq = 0 gives nothing.  Raises
    FormatError where the engine must refuse the stream (cap: the longest record a batch takes, when given)."""
    n = len(stream)
    if n < 8:
        raise FormatError(0, "Truncated BAM header")
    if stream[:4] != b"BAM\1":
        raise FormatError(0, "Invalid BAM magic")
    at = 8 + _le32(stream, 4)
    if at + 4 > n:
        raise FormatError(0, "Truncated BAM header")
    n_ref = struct.unpack_from("<i", stream, at)[0]
    if n_ref < 0:
        raise FormatError(at, "Invalid BAM header: negative number of references")
    at += 4
    for _ in range(n_ref):
        if at + 4 > n:
            raise FormatError(at, "Truncated BAM header")
        at += 4 + _le32(stream, at) + 4
        if at > n:
            raise FormatError(at, "Truncated BAM header")
    out = []
    while at < n:
        if at + 4 > n:
            raise FormatError(at, "Truncated BAM record")
        bs = _le32(stream, at)
        if bs < 32:
            raise FormatError(at, "block_size %d is below the 32 bytes of its fixed fields" % bs)
        if cap is not None and 4 + bs > cap:
            raise FormatError(at, "longer than the staging buffer")
        if at + 4 + bs > n:
            raise FormatError(at, "Truncated BAM record")
        l_name, n_cigar = stream[at + 12], struct.unpack_from("<H", stream, at + 16)[0]
        l_seq = struct.unpack_from("<i", stream, at + 20)[0]
        s = 36 + l_name + 4 * n_cigar
        q = s + (l_seq + 1) // 2
        if l_seq < 0 or q + l_seq > 4 + bs:
            raise FormatError(at, "its fields run past its block_size")
        if l_seq:
            packed = stream[at + s:at + q]
            codes = [packed[j // 2] >> 4 if j % 2 == 0 else packed[j // 2] & 15 for j in range(l_seq)]
            seq = bytes(b"NACNGNNNTNNNNNNN"[c] for c in codes)
            qual = bytes((c + 33) & 0xff for c in stream[at + q:at + q + l_seq])
            out.append((at, b"@\n" + seq + b"\n+\n" + qual + b"\n"))
        at += 4 + bs
    return out


def bam_model_fastq(stream, cap=None):
    return b"".join(r for _, r in bam_model_records(stream, cap))


# ---- batch walks ---------------------------------------------------------------------------------------------------------
def sam_caps(max_batch_bytes):
    """(in_cap, cap) of an engine whose table is small enough that the record pool is off: the scratch capacity of the
    transcode and the most input bytes of one batch (jf_engine.cu, sam_alloc and sam_batch_cap)."""
    bb = (max_batch_bytes + 15) & ~15 if max_batch_bytes else 64 << 20
    in_cap = max(min(bb // 2, 1 << 30) & ~15, 64)
    return in_cap, max(in_cap & ~15, 16)


class Batch(object):
    """One transcode launch: bytes [off, off + n) of the file at lo = the first byte's offset from A; `used` = the bytes it
    consumes (through its last newline, or all of them in the file's last batch)."""

    def __init__(self, off, lo, n, used):
        self.off, self.lo, self.n, self.used = off, lo, n, used
        self.hi = lo + n
        self.tiles = -(-self.hi // TILE)

    def rel(self, pos):
        """offset from A of file byte pos"""
        return pos - self.off + self.lo

    def __repr__(self):
        return "Batch(off=%d, lo=%d, hi=%d, tiles=%d)" % (self.off, self.lo, self.hi, self.tiles)


class TooLong(Exception):
    pass


def host_walk(data, cap):
    """The batches of SAM text fed from host memory in one call: each ends at the last newline at or before `cap` bytes, the
    last takes the rest.  A host batch is staged at an aligned buffer: lo = 0."""
    out, pos, n = [], 0, len(data)
    while pos < n:
        ln = min(cap, n - pos)
        if pos + ln < n:
            nl = data.rfind(b"\n", pos, pos + ln)
            if nl < 0:
                raise TooLong(pos)
            ln = nl + 1 - pos
        out.append(Batch(pos, 0, ln, ln))
        pos += ln
    return out


def device_walk(data, cap, base=0):
    """The batches of SAM text fed from device memory at an address `base` bytes past a 16-byte boundary, in one call: each
    takes `cap` bytes (or the rest) and consumes them through its last newline; the next starts there."""
    out, pos, n = [], 0, len(data)
    while pos < n:
        ln = min(cap, n - pos)
        if pos + ln == n:
            used = ln
        else:
            used = data.rfind(b"\n", pos, pos + ln) + 1 - pos
            if used <= 0:
                raise TooLong(pos)
        out.append(Batch(pos, (base + pos) & 15, ln, used))
        pos += used
    return out


def line_starts(data):
    """offsets of the record lines: not headers ('@'), not blank ("\\n" or "\\r\\n")"""
    out, at = [], 0
    parts = data.split(b"\n")
    for j, ln in enumerate(parts):
        if ln and ln[:1] != b"@" and not (ln == b"\r" and j + 1 < len(parts)):
            out.append(at)
        at += len(ln) + 1
    return out


def batch_of(walk, pos):
    for i, b in enumerate(walk):
        if b.off <= pos < b.off + b.used:
            return i, b
    raise IndexError(pos)


def where(walk, pos):
    """pos's batch and its place relative to that batch's A, word and tile"""
    i, b = batch_of(walk, pos)
    r = b.rel(pos)
    return "batch %d %r: A + %d, word %d byte %d, tile %d byte %d" % (i, b, r, r // WORD, r % WORD, r // TILE, r % TILE)


def first_mismatch(got, records, walk=None):
    """None, or a message naming the first output byte that differs from the model's records [(line offset, FASTQ)]"""
    want = b"".join(r for _, r in records)
    if got == want:
        return None
    i = next((j for j in range(min(len(got), len(want))) if got[j] != want[j]), min(len(got), len(want)))
    at, ri = 0, 0
    while ri < len(records) and at + len(records[ri][1]) <= i:
        at += len(records[ri][1])
        ri += 1
    msg = "output %d bytes, model %d; first difference at output byte %d" % (len(got), len(want), i)
    if ri < len(records):
        line = records[ri][0]
        msg += " (byte %d of record %d, the line at file byte %d%s): got %r, want %r" % (
            i - at, ri, line, "; " + where(walk, line) if walk else "", got[at:at + len(records[ri][1])][:80], records[ri][1][:80])
    return msg


# ---- the aimed SAM cells -------------------------------------------------------------------------------------------------
def rec(name, seq, qual, tags=b"", eol=b"\n", flag=b"0"):
    return b"\t".join([name, flag, b"chr1", b"1", b"60", b"*", b"*", b"0", b"0", seq, qual]) + tags + eol


def _bases(n, i, alphabet=b"ACGT"):
    return bytes(alphabet[(i * 7 + j * 5 + j * j) % len(alphabet)] for j in range(n))


def _qual(n, i):
    return bytes(33 + (i * 3 + j * 11) % 42 for j in range(n))


def corpus_block():
    """The cell lines, each with QNAME lengths 1 ... 32 so that its tabs, '\\r' and '\\n' take every lane of the stride."""
    lines = []
    for L in range(1, 33):
        nm = b"q" * L
        lines += [
            rec(nm, _bases(3, L), _qual(3, L)),                                   # exactly 10 tabs; the next line in the stride
            rec(nm, _bases(5, L), _qual(5, L), tags=b"\tXA:Z:"),                   # tab 11 and '\n' in one stride
            rec(nm, _bases(4, L), _qual(4, L), eol=b"\r\n"),                      # '\r' and '\n' through every lane
            rec(nm, _bases(6, L), b"*", eol=b"\r\n"),                             # QUAL '*' with "\r\n"
            rec(nm, b"*", b"*", tags=b"\tNM:i:0"),                                # no bases
            b"\t" * 9 + _bases(L % 5 + 1, L) + b"\t" + _qual(L % 5 + 1, L) + b"\n",  # empty fields
            rec(nm, _bases(40 + L, L, b"ACGTacgtNRYKM=.U"), _qual(40 + L, L)),   # IUPAC and lower case, over two strides
            b"\n" if L % 2 else b"\r\n",                                          # blank lines
            b"@CO\t" + b"c" * (L - 1) + b"\n",                                    # a header line among the records
        ]
    return b"".join(lines)


def pad(p):
    """p bytes of header lines of at most 32 bytes ('\\n' alone for 1 byte)"""
    out = [b"@" + b"x" * 30 + b"\n"] * (p // 32)
    r = p % 32
    out.append(b"" if r == 0 else b"\n" if r == 1 else b"@" + b"x" * (r - 2) + b"\n")
    return b"".join(out)


def padded(p, block, final_newline=True):
    """p bytes of header in front of the block; without a final newline the block's last record line is cut short of it"""
    body = block
    if not final_newline:
        body = body.rstrip(b"\n")
        body = body[:body.rfind(b"\n") + 1] + rec(b"last", b"ACGT", b"IIII")[:-1]
    return pad(p) + body


def tile_pads(block, every=1):
    """header lengths that put a newline of the block at the last byte of a tile, one byte before, and one after"""
    nls = [i for i, c in enumerate(block) if c == 10][::every]
    return sorted({TILE - 1 - x + d for x in nls for d in (-1, 0, 1) if TILE - 1 - x + d >= 0})


# ---- large fixed-width SAM -----------------------------------------------------------------------------------------------
def kinds(n, zero_every=0, crlf_every=0, star_qual_every=0):
    """masks of the lines with SEQ '*' and QUAL '*', with "\\r\\n", with QUAL '*' (not with a '*' SEQ)"""
    i = np.arange(n)
    zero = i % zero_every == zero_every - 1 if zero_every else np.zeros(n, bool)
    crlf = i % crlf_every == 1 if crlf_every else np.zeros(n, bool)
    sq = (i % star_qual_every == 2) & ~zero if star_qual_every else np.zeros(n, bool)
    return zero, crlf, sq


def fixed_lines(xp, seq, qual, width, zero, crlf, sq, mids=(b"\t" * 9,), tail=b""):
    """(n, width) SAM lines, QNAME (all 'q') padding each to `width`: QNAME, mids[i % len(mids)] (the tab behind QNAME
    through the tab in front of SEQ), SEQ, tab, QUAL, `tail` (tags), [\\r] \\n.  xp is numpy or torch; seq and qual are (n, R)
    uint8 arrays of it, the masks bool arrays of it (see kinds)."""
    n, R = seq.shape
    dev = {} if xp is np else {"device": seq.device}
    lines = xp.full((n, width), ord("q"), dtype=xp.uint8, **dev)
    assert width >= 1 + max(len(m) for m in mids) + 2 * R + 2 + len(tail)
    which = xp.arange(n, **dev) % len(mids)
    for v, mid in enumerate(mids):
        mv = np.frombuffer(mid, np.uint8) if xp is np else xp.frombuffer(bytearray(mid), dtype=xp.uint8).to(seq.device)
        tv = np.frombuffer(tail, np.uint8) if xp is np else xp.frombuffer(bytearray(tail or b"x"), dtype=xp.uint8).to(seq.device)
        for z in (0, 1):
            for c in (0, 1):
                for s in (0, 1):
                    m = (which == v) & (zero == bool(z)) & (crlf == bool(c)) & (sq == bool(s))
                    if z and s or not bool(m.any()):
                        continue
                    end = width - 1 - c
                    lines[m, width - 1] = 10
                    if c:
                        lines[m, width - 2] = 13
                    if tail:
                        lines[m, end - len(tail):end] = tv
                    qe = end - len(tail)
                    q0 = qe - 1 if z or s else qe - R
                    if z or s:
                        lines[m, q0] = ord("*")
                    else:
                        lines[m, q0:qe] = qual[m]
                    lines[m, q0 - 1] = 9
                    s0 = q0 - 2 if z else q0 - 1 - R
                    if z:
                        lines[m, s0] = ord("*")
                    else:
                        lines[m, s0:q0 - 1] = seq[m]
                    lines[m, s0 - len(mid):s0] = mv
    return lines


def fixed_fields(xp, lines, R, crlf, sq, tail=b""):
    """(seq, qual) read back from the columns where fixed_lines put them (lines without a '*' SEQ; the qual of a QUAL '*'
    line is junk, which fixed_fastq replaces)"""
    n, width = lines.shape
    dev = {} if xp is np else {"device": lines.device}
    seq = xp.empty((n, R), dtype=xp.uint8, **dev)
    qual = xp.empty((n, R), dtype=xp.uint8, **dev)
    for c in (0, 1):
        for s in (0, 1):
            m = (crlf == bool(c)) & (sq == bool(s))
            qe = width - 1 - c - len(tail)
            q0 = qe - 1 if s else qe - R
            seq[m] = lines[m, q0 - 1 - R:q0 - 1]
            qual[m] = lines[m, qe - R:qe]
    return seq, qual


def fixed_fastq(xp, seq, qual, zero, sq):
    """the FASTQ of fixed_lines as an (m, 2 R + 6) array: one row per line that has bases"""
    keep = ~zero
    s, q, star = seq[keep], qual[keep], sq[keep]
    m, R = s.shape
    fq = xp.empty((m, 2 * R + 6), dtype=xp.uint8) if xp is np else xp.empty((m, 2 * R + 6), dtype=xp.uint8, device=seq.device)
    fq[:, 0], fq[:, 1] = ord("@"), 10
    fq[:, 2:2 + R] = s
    fq[:, 2 + R], fq[:, 3 + R], fq[:, 4 + R] = 10, ord("+"), 10
    fq[:, 5 + R:5 + 2 * R] = q
    fq[star, 5 + R:5 + 2 * R] = 32
    fq[:, -1] = 10
    return fq


def fixed_sam(n, read_len, width=None, head=0, seed=1, **kw):
    """n fixed-width lines (fixed_lines, random bases and qualities) behind `head` bytes of header lines, with numpy ->
    (sam bytes, FASTQ bytes, width)"""
    rng = np.random.default_rng(seed)
    seq = np.frombuffer(b"ACGT", np.uint8)[rng.integers(0, 4, (n, read_len))]
    qual = rng.integers(43, 75, (n, read_len), dtype=np.uint8)     # (no "*": a one-base QUAL "*" means no qualities)
    zero, crlf, sq = kinds(n, **kw)
    width = width or 9 + 2 * read_len + 3 + int(crlf.any())
    lines = fixed_lines(np, seq, qual, width, zero, crlf, sq)
    return pad(head) + lines.tobytes(), fixed_fastq(np, seq, qual, zero, sq).tobytes(), width
