"""SAM and BAM writers made from the SAM specification (v1.6, sections 1.4, 4.1 and 4.2), and a model of what `count --sam`
reads from a SAM file.  Nothing here comes from the reference's fastq2sam.cc.

* fastq_to_sam: 4-line FASTQ -> SAM with realistic fields (FLAG 0 / 4 / 16 / 256, CIGAR, optional tags).
* sam_to_bam:   SAM -> the uncompressed BAM stream (magic, header text, references, records).
* bgzf:         BGZF blocks of a byte stream, cut at fixed sizes so records straddle blocks, and the end-of-file block.
* sam_model_fastq: the FASTQ the engine must count for a SAM file -- one "@\\n SEQ \\n+\\n QUAL \\n" record per alignment.
"""
import re
import struct
import zlib

FLAGS = (0, 4, 16, 256)


def parse_fastq(data):
    lines = data.split(b"\n")
    return [(lines[i][1:], lines[i + 1], lines[i + 3]) for i in range(0, len(lines) - 3, 4)]


def fastq_to_sam(data, ref_len=1000000):
    out = [b"@HD\tVN:1.6\tSO:unsorted\n", b"@SQ\tSN:chr1\tLN:%d\n" % ref_len, b"@SQ\tSN:chr2\tLN:5000\n",
           b"@RG\tID:grp1\tSM:sample\n", b"@PG\tID:writer\tPN:sam_tools\n"]
    for i, (name, seq, qual) in enumerate(parse_fastq(data)):
        flag = FLAGS[i % 4]
        unmapped = flag & 4
        rname, pos, mapq = (b"*", 0, 0) if unmapped else (b"chr1", 1 + (i * 37) % ref_len, 60)
        cigar = b"*" if unmapped or not seq else (b"%dM" % len(seq) if i % 3 else b"2S%dM" % (len(seq) - 2) if len(seq) > 2 else b"%dM" % len(seq))
        out.append(b"\t".join([name.split()[0] or b"r%d" % i, b"%d" % flag, rname, b"%d" % pos, b"%d" % mapq, cigar, b"*", b"0", b"0",
                               seq or b"*", qual or b"*", b"NM:i:%d" % (i % 5), b"RG:Z:grp1", b"AS:i:%d" % (len(seq) - i % 7)]) + b"\n")
    return b"".join(out)


_CIGAR_OPS = b"MIDNSHP=X"
_NT16 = "=ACMGRSVTWYHKDBN"


def _tag(t):
    tag, typ, val = t.split(b":", 2)
    if typ == b"i":
        return tag + b"i" + struct.pack("<i", int(val))
    return tag + b"Z" + val + b"\0"


def sam_to_bam(sam):
    """The uncompressed BAM stream of a SAM file (SAM specification 4.2)."""
    header, refs, recs = [], [], []
    for line in sam.split(b"\n"):
        if not line:
            continue
        if line.startswith(b"@"):
            header.append(line + b"\n")
            m = re.match(rb"@SQ\tSN:(\S+)\tLN:(\d+)", line)
            if m:
                refs.append((m.group(1), int(m.group(2))))
            continue
        f = line.split(b"\t")
        names = [r[0] for r in refs]
        ref_id = names.index(f[2]) if f[2] in names else -1
        seq = b"" if f[9] == b"*" else f[9]
        qual = bytes([0xff] * len(seq)) if f[10] == b"*" else bytes(c - 33 for c in f[10])
        cig = [] if f[5] == b"*" else [(int(n), _CIGAR_OPS.index(op)) for n, op in re.findall(rb"(\d+)([MIDNSHP=X])", f[5])]
        name = f[0] + b"\0"
        codes = [_NT16.find(chr(c).upper()) for c in seq]
        codes = [c if c >= 0 else 15 for c in codes] + [0]
        packed = bytes(codes[i] << 4 | codes[i + 1] for i in range(0, len(seq), 2))
        body = struct.pack("<iiBBHHHiiii", ref_id, int(f[3]) - 1, len(name), int(f[4]), 4680, len(cig), int(f[1]), len(seq),
                           -1, -1, 0)
        body += name + b"".join(struct.pack("<I", n << 4 | op) for n, op in cig) + packed + qual + b"".join(_tag(t) for t in f[11:])
        recs.append(struct.pack("<I", len(body)) + body)
    text = b"".join(header)
    out = b"BAM\1" + struct.pack("<i", len(text)) + text + struct.pack("<i", len(refs))
    for name, ln in refs:
        out += struct.pack("<i", len(name) + 1) + name + b"\0" + struct.pack("<i", ln)
    return out + b"".join(recs)


def bgzf_block(data):
    c = zlib.compressobj(6, zlib.DEFLATED, -15)
    cdata = c.compress(data) + c.flush()
    bsize = 18 + len(cdata) + 8 - 1
    head = b"\x1f\x8b\x08\x04\x00\x00\x00\x00\x00\xff" + struct.pack("<HBBHH", 6, ord("B"), ord("C"), 2, bsize)
    return head + cdata + struct.pack("<II", zlib.crc32(data), len(data))


BGZF_EOF = bgzf_block(b"")


def bgzf(data, block=65280):
    """BGZF of `data` cut every `block` bytes (records straddle blocks), then the end-of-file block."""
    return b"".join(bgzf_block(data[i:i + block]) for i in range(0, len(data), block)) + BGZF_EOF


class FormatError(ValueError):
    """Where the engine must refuse a file: `offset` is the byte of the file the engine's message names, `what` the reason
    it gives."""

    def __init__(self, offset, what):
        super().__init__("%s (at byte %d)" % (what, offset))
        self.offset, self.what = offset, what


def sam_model_records(sam):
    """[(byte offset of the line, its FASTQ record)] for the SAM lines that give bases; see sam_model_fastq."""
    out = []
    lines = sam.split(b"\n")
    last = lines.pop()                       # (b"" when the file ends with a newline)
    lines = [ln[:-1] if ln.endswith(b"\r") else ln for ln in lines] + ([last] if last else [])
    at = 0
    for ln, raw in zip(lines, sam.split(b"\n")):
        start, at = at, at + len(raw) + 1
        if not ln or ln.startswith(b"@"):
            continue
        f = ln.split(b"\t")
        if len(f) < 11:
            raise FormatError(start, "fewer than 11 fields")
        seq = b"" if f[9] == b"*" else f[9]
        if f[10] == b"*":
            qual = b" " * len(seq)
        elif len(f[10]) != len(seq):
            raise FormatError(start, "SEQ and QUAL of different lengths")
        else:
            qual = f[10]
        if seq:
            seq = bytes(c if c in b"ACGTacgt" else ord("N") for c in seq)
            out.append((start, b"@\n" + seq + b"\n+\n" + qual + b"\n"))
    return out


def sam_model_fastq(sam):
    """The FASTQ `count --sam` counts for a SAM file: header ('@') and blank lines skipped, one '\\r' before a '\\n' dropped,
    SEQ field 10 and QUAL field 11, a '*' SEQ gives no bases, a '*' QUAL gives every base the quality character 0x20, bytes
    other than ACGTacgt become N.  Raises FormatError (a ValueError) with the offset of the first bad line where the engine
    must refuse the file."""
    return b"".join(r for _, r in sam_model_records(sam))
