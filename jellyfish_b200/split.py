"""Split one FASTA or FASTQ file among the ranks of a multi-GPU count (pure Python, no device).

Rank r of N owns the bytes [s_r, s_{r+1}) of a file of S bytes, s_0 = 0 and s_N = S.  Every rank computes the cuts it needs
from a few small windows of the file around the nominal cut a_r = r * S // N, so no cut is communicated.  The cuts are
monotone: a rank whose share is empty (s_r >= s_{r+1}, e.g. a file of fewer lines than ranks) counts nothing.

FASTA: s_r is the first line start >= a_r.  A line start is parser state L, so the share can be parsed from there as a
continuation (JFGPU_FORMAT_FASTA).  What the share's first k-mers need from the text in front of it -- the last k - 1
symbols -- comes from the seam [c_r, s_r): whole lines walked back from s_r up to the start of a header line, the file
start, or until they hold k - 1 bytes of ACGTacgt.  Each line is parsed the same way wherever the parse starts, and a
non-base byte is a reset, which only shortens what must be carried; so parsing [c_r, s_r) (jfgpu_seam) leaves exactly the
symbols a parse of the whole file carries into s_r.  A share that starts on a header line needs no seam.  The seam is
read whole: for FASTA whose sequences are not wrapped it is the whole sequence line in front of the cut.

Under -Q (`headers=True`) a FASTA share starts on a header line instead: s_r is the first line start >= a_r whose first
byte is '>'.  The parser with -Q reads '\r' by other rules than the seam knows (include/jfgpu.h, jfgpu_seam), and a share
that starts on a header needs no seam.  A file of fewer records than ranks, or one whose records are few and long (a
genome of a few chromosomes), then leaves some ranks an empty or a short share: the count is the same, only fewer GPUs
parse it.

FASTQ (4-line records): s_r is the first line start >= a_r where two consecutive records look whole ('@' line, a line,
'+' line, a line as long as the sequence line).  Every read starts with a reset, so there is no seam.  This local rule is
not exact -- a sequence line may start with '@' and a quality line with '+' -- so the caller checks every cut afterwards:
the number of lines in front of s_r must be a multiple of 4 (`fastq_cuts_ok`).

Only text is split: gzip and other inputs are refused by `sniff`, as the multi-GPU commands refuse them.
"""
import collections
import os
import stat

WINDOW = 1 << 16          # bytes read at a time while looking for a cut

Share = collections.namedtuple("Share", "fmt seam start end")
Share.__doc__ = """Rank r's part of a file: parse [seam, start) without counting it (FASTA only; seam == start when there is
no seam), then count [start, end).  fmt: "fasta" or "fastq"."""


def sniff(first_byte):
    """The format the engine reads a file in, from its first byte: "fasta", "fastq", None for an empty file; ValueError for
    anything else (mer_overlap_sequence_parser.hpp:134-148)."""
    if not first_byte:
        return None
    if first_byte[:1] == b">":
        return "fasta"
    if first_byte[:1] == b"@":
        return "fastq"
    raise ValueError("Unsupported format")


def splittable(path):
    """True for a regular file, which can be read at any offset.  A pipe or a process substitution (`<(zcat reads.fq.gz)`)
    can be read once, from its start: the caller gives it whole to one rank."""
    try:
        return stat.S_ISREG(os.stat(path).st_mode)
    except OSError:
        return False


def _line_start_at_or_after(read, size, a):
    """The first line start >= a (size when there is none)."""
    if a <= 0:
        return 0
    p = a - 1                 # the line starting at a needs a '\n' at a - 1
    while p < size:
        w = read(p, min(WINDOW, size - p))
        i = w.find(b"\n")
        if i >= 0:
            return p + i + 1
        p += len(w)
    return size


def _line_before(read, end):
    """The line that ends right in front of the line start `end` (end > 0) -> (start, bytes without its '\\n')."""
    stop = end - 1            # read[end - 1] is the '\n' ending the line
    chunks = []
    p = stop
    while p > 0:
        lo = max(0, p - WINDOW)
        w = read(lo, p - lo)
        i = w.rfind(b"\n")
        if i >= 0:
            chunks.append(w[i + 1:])
            start = lo + i + 1
            break
        chunks.append(w)
        p = lo
    else:
        start = 0
    return start, b"".join(reversed(chunks))


def fasta_seam_start(read, start, k):
    """c: where the seam in front of the line start `start` begins (see the module documentation)."""
    c, need = start, k - 1
    if start > 0 and read(start, WINDOW).lstrip(b"\r")[:1] == b">":
        return start          # a header line resets the window: nothing in front of it matters
    while c > 0 and need > 0:
        c, line = _line_before(read, c)
        if line.lstrip(b"\r")[:1] == b">":
            break
        need -= len(line) - len(line.translate(None, b"ACGTacgt"))
    return c


def fasta_header_at_or_after(read, size, a):
    """The first line start >= a whose first byte is '>' (size when there is none)."""
    if a <= 0:
        return 0
    p = a - 1                 # a header at q needs a '\n' at q - 1
    while p < size:
        w = read(p, min(WINDOW, size - p))
        i = w.find(b"\n>")
        if i >= 0:
            return p + i + 1
        if p + len(w) >= size:
            break
        p += len(w) - 1       # (the windows overlap by one byte: a "\n>" across two is found)
    return size


def _lines_from(read, size, p, n):
    """Up to n lines starting at the line start p -> list of (start, bytes without the '\\n')."""
    w = WINDOW
    while True:
        buf = read(p, min(w, size - p))
        parts = buf.split(b"\n")
        at_eof = p + len(buf) >= size
        if len(parts) > n or at_eof:
            break
        w *= 2
    lines = parts[:-1] + ([parts[-1]] if at_eof and parts[-1] else [])
    out = []
    for line in lines[:n]:
        out.append((p, line))
        p += len(line) + 1
    return out


def _fastq_looks_whole(lines):
    if len(lines) < 8:
        return False
    for r in (0, 4):
        hdr, sq, plus, q = (lines[r + j][1] for j in range(4))
        if hdr[:1] != b"@" or plus[:1] != b"+" or len(q) != len(sq):
            return False
    return True


def fastq_share_start(read, size, a):
    """The first line start >= a where two consecutive records look whole (size when there is none)."""
    p = _line_start_at_or_after(read, size, a)
    while p < size:
        lines = _lines_from(read, size, p, 9)
        if _fastq_looks_whole(lines):
            return p
        if len(lines) < 2:
            return size
        p = lines[1][0]
    return size


def share_start(read, size, fmt, a, headers=False):
    """s for the nominal cut a (0 -> 0).  headers: FASTA shares start on header lines (-Q)."""
    if a <= 0:
        return 0
    if fmt == "fasta":
        return fasta_header_at_or_after(read, size, a) if headers else _line_start_at_or_after(read, size, a)
    return fastq_share_start(read, size, a)


def plan_share(read, size, fmt, rank, world, k, headers=False):
    """Share of `rank` in a file of `size` bytes read through read(offset, n) -> bytes.  headers=True (-Q): a FASTA share
    starts on a header line and has no seam."""
    s = share_start(read, size, fmt, rank * size // world, headers)
    e = size if rank == world - 1 else share_start(read, size, fmt, (rank + 1) * size // world, headers)
    e = max(e, s)
    seam = fasta_seam_start(read, s, k) if fmt == "fasta" and s < e and not headers else s
    return Share(fmt, seam, s, e)


def plan_file(path, rank, world, k, headers=False):
    """plan_share of a regular file (pread; see `splittable`); None for an empty file.  ValueError: not FASTA or FASTQ
    text."""
    fd = os.open(path, os.O_RDONLY)
    try:
        size = os.fstat(fd).st_size
        fmt = sniff(os.pread(fd, 1, 0))
        if fmt is None:
            return None
        return plan_share(lambda off, n: os.pread(fd, n, off), size, fmt, rank, world, k, headers)
    finally:
        os.close(fd)


def fastq_cuts_ok(tallies):
    """tallies[r] = (bytes, newlines) of rank r's share of a FASTQ file, in rank order.  True when every share that is not
    empty starts on a record, i.e. behind a multiple of 4 lines."""
    at = 0
    for n_bytes, newlines in tallies:
        if n_bytes and at % 4:
            return False
        at += newlines
    return True
