"""Split one SAM or BAM file among the ranks of a multi-GPU count (pure Python, no device), as split.py splits FASTA and
FASTQ: every rank computes its own cuts from a few small windows of the file, and no cut is communicated.

SAM text: rank r of N counts the lines from the first line start at or after r * S // N up to where rank r + 1's share
starts.  Header lines start with '@' and are skipped wherever they are, and a QNAME cannot start with '@', so every line
start is a record boundary: the cuts are exact and need no check.

BAM (BGZF, SAM specification 4.1 and 4.2): a position in the file is a pair (block, offset) -- the byte offset of a BGZF
block in the file and an offset into its inflated data.  Rank r's block cut c_r is the first BGZF block header at or after
r * S // N whose BSIZE chain is followed through CHAIN blocks (or to the end of the file).  Its record cut is the first
position at or after (c_r, 0) where CHAIN records in a row parse consistently: block_size >= 32, refID and next_refID in
[-1, n_ref), l_read_name >= 1 with a NUL at its end, l_seq >= 0, and the name, CIGAR, SEQ and QUAL inside block_size.
n_ref comes from the header, which every rank reads from the start of the file.  Rank 0 starts at the file start, header
included.  A rank counts the records from its cut up to the next rank's cut, reading past its last block when its last
record runs on.  That rule can be fooled (tags may hold bytes that look like records), so the caller checks every cut
afterwards: the record chain of rank r, followed from its cut, must end exactly at rank r + 1's cut -- the engine reports a
record cut short there -- and when it does not, every rank counts whole files instead.  Rank 0's cut is exact, so a chain
that meets every next cut is the file's own chain.

gzip'd SAM (BGZF-compressed SAM included) cannot be split: `kind` tells it apart and the caller counts it whole.
"""
import collections
import os
import struct
import zlib

from .split import WINDOW, _line_start_at_or_after

BGZF_HEAD = 18            # bytes of a BGZF block header: gzip header with the one extra subfield "BC" (BSIZE)
BGZF_MIN = 28             # header, the shortest deflate stream, CRC32 and ISIZE
CHAIN = 4                 # BGZF blocks, and BAM records, that must follow a cut for it to be taken
EMPTY_BAM_HEADER = b"BAM\1" + struct.pack("<ii", 0, 0)     # what the engine reads in front of a share that starts at a record

BamShare = collections.namedtuple("BamShare", "start end")
BamShare.__doc__ = """Rank r's part of a BAM file: the records from `start` up to `end`, both (block offset, offset into the
block's inflated data); (file size, 0) is the end of the file.  start == (0, 0): the share begins with the header."""


def kind(path):
    """'sam', 'bam', 'gz' (gzip'd SAM, BGZF-compressed SAM included: not splittable), 'cram', or None for an empty file --
    from the first bytes of a regular file."""
    with open(path, "rb") as f:
        head = f.read(BGZF_HEAD)
        if not head:
            return None
        if head.startswith(b"CRAM"):
            return "cram"
        if head[:2] != b"\x1f\x8b":
            return "sam"
        bs = block_size(head)
        if bs is None:
            return "gz"
        f.seek(0)
        data = inflate_block(f.read(bs), 0)
        return "bam" if data[:4] == b"BAM\1" else "gz"


def block_size(head):
    """BSIZE + 1 of the BGZF block whose header is `head` (at least 18 bytes), None when it is not a BGZF header."""
    if len(head) < BGZF_HEAD or head[:4] != b"\x1f\x8b\x08\x04" or head[10:16] != b"\x06\x00BC\x02\x00":
        return None
    return struct.unpack_from("<H", head, 16)[0] + 1


def inflate_block(raw, at):
    """The data of the whole BGZF block `raw`, which starts at byte `at` of the file.  ValueError for a block that is cut
    short or corrupt (its deflate stream, CRC32 or ISIZE)."""
    bs = block_size(raw)
    if bs is None or len(raw) != bs or bs < BGZF_MIN:
        raise ValueError("corrupt or truncated BGZF block at byte %d" % at)
    crc, isize = struct.unpack_from("<II", raw, bs - 8)
    try:
        data = zlib.decompress(raw[BGZF_HEAD:bs - 8], -15)
    except zlib.error as ex:
        raise ValueError("corrupt BGZF block at byte %d: %s" % (at, ex))
    if len(data) != isize or zlib.crc32(data) != crc:
        raise ValueError("corrupt BGZF block at byte %d: CRC32 or ISIZE does not match its data" % at)
    return data


def _blocks_follow(read, size, p, n=CHAIN):
    """True when n BGZF blocks follow one another from p, or the blocks from p reach the end of the file exactly."""
    for _ in range(n):
        if p == size:
            return True
        bs = block_size(read(p, BGZF_HEAD))
        if bs is None or bs < BGZF_MIN or p + bs > size:
            return False
        p += bs
    return True


def block_cut(read, size, a):
    """The first BGZF block at or after byte a whose BSIZE chain holds (size when there is none)."""
    if a <= 0:
        return 0
    p = a
    while p < size:
        w = read(p, min(WINDOW, size - p) + 3)
        i = w.find(b"\x1f\x8b\x08\x04")
        while i >= 0:
            if _blocks_follow(read, size, p + i):
                return p + i
            i = w.find(b"\x1f\x8b\x08\x04", i + 1)
        p += max(1, len(w) - 3)
    return size


def walk_blocks(read, size, p, stop):
    """[(offset, bsize, isize)] of the blocks from the block start p up to the first block at or after `stop`, excluded.
    ValueError when the chain breaks (a block cut short or not a BGZF block)."""
    out = []
    buf, base = b"", p
    while p < stop:
        if p + BGZF_HEAD > base + len(buf):
            buf, base = read(p, 16 * WINDOW), p
        bs = block_size(buf[p - base:p - base + BGZF_HEAD])
        if bs is None or bs < BGZF_MIN or p + bs > size:
            raise ValueError("corrupt or truncated BGZF block at byte %d" % p)
        if p + bs > base + len(buf):
            buf, base = read(p, max(16 * WINDOW, bs)), p
        out.append((p, bs, struct.unpack_from("<I", buf, p - base + bs - 4)[0]))
        p += bs
    return out


class _Inflated(object):
    """The inflated stream of the blocks from block start p, inflated as far as it is asked for."""

    def __init__(self, read, size, p):
        self.read, self.size, self.next = read, size, p
        self.data = bytearray()
        self.starts = []                  # (block offset, offset of its data in self.data)

    def ensure(self, n):
        """True when the stream holds at least n bytes; False when the file ends first."""
        while len(self.data) < n:
            if self.next >= self.size:
                return False
            bs = block_size(self.read(self.next, BGZF_HEAD))
            if bs is None or self.next + bs > self.size:
                raise ValueError("corrupt or truncated BGZF block at byte %d" % self.next)
            self.starts.append((self.next, len(self.data)))
            self.data += inflate_block(self.read(self.next, bs), self.next)
            self.next += bs
        return True

    def position(self, o):
        """(block, offset) of stream offset o (the block that holds byte o; (size, 0) at the end of the file)."""
        if not self.ensure(o + 1):
            return (self.size, 0)
        for b, s in reversed(self.starts):
            if s <= o:
                return (b, o - s)


def bam_header(read, size):
    """-> (n_ref, bytes of the header: magic, text and references) of a BAM file.  ValueError for a bad magic or a cut."""
    s = _Inflated(read, size, 0)
    if not s.ensure(12) or bytes(s.data[:4]) != b"BAM\1":
        raise ValueError("Invalid BAM magic")
    o = 8 + struct.unpack_from("<i", s.data, 4)[0]
    if not s.ensure(o + 4):
        raise ValueError("Truncated BAM header")
    n_ref = struct.unpack_from("<i", s.data, o)[0]
    o += 4
    for _ in range(n_ref):
        if not s.ensure(o + 4):
            raise ValueError("Truncated BAM header")
        o += 8 + struct.unpack_from("<i", s.data, o)[0]
    if not s.ensure(o) and o != len(s.data):
        raise ValueError("Truncated BAM header")
    return n_ref, o


def records_follow(s, o, n_ref, n=CHAIN):
    """True when n records in a row parse consistently from stream offset o (see the module documentation), or the records
    from o reach the end of the file exactly."""
    for _ in range(n):
        if not s.ensure(o + 36):
            return o == len(s.data)
        bsz, ref, _, l_name, _, _, n_cig, _, l_seq, nref = struct.unpack_from("<IiiBBHHHii", s.data, o)
        if bsz < 32 or not -1 <= ref < n_ref or not -1 <= nref < n_ref or l_name < 1 or l_seq < 0:
            return False
        if 32 + l_name + 4 * n_cig + (l_seq + 1) // 2 + l_seq > bsz:
            return False
        if not s.ensure(o + 36 + l_name) or s.data[o + 35 + l_name] != 0:
            return False
        o += 4 + bsz
    return True


def record_cut(read, size, n_ref, c):
    """The first position at or after (c, 0) where CHAIN records parse consistently ((size, 0) when there is none)."""
    s = _Inflated(read, size, c)
    o = 0
    while s.ensure(o + 1):
        if records_follow(s, o, n_ref):
            return s.position(o)
        o += 1
    return (size, 0)


def bam_share_start(read, size, n_ref, header_end, a):
    """Where the share of the nominal cut a starts: (0, 0) for a = 0, else the record cut behind the block cut of a, and
    never inside the header."""
    if a <= 0:
        return (0, 0)
    c = block_cut(read, size, a)
    if c >= size:
        return (size, 0)
    return max(record_cut(read, size, n_ref, c), header_end)


def plan_bam_share(read, size, rank, world):
    """BamShare of `rank` in a BAM file of `size` bytes read through read(offset, n) -> bytes."""
    n_ref, hlen = bam_header(read, size)
    header_end = _Inflated(read, size, 0).position(hlen) if hlen else (0, 0)
    start = bam_share_start(read, size, n_ref, header_end, rank * size // world)
    end = (size, 0) if rank == world - 1 else bam_share_start(read, size, n_ref, header_end, (rank + 1) * size // world)
    return BamShare(start, max(start, end))


def plan_sam_share(read, size, rank, world):
    """(start, end) of `rank`'s lines of a SAM text file."""
    s = _line_start_at_or_after(read, size, rank * size // world)
    e = size if rank == world - 1 else _line_start_at_or_after(read, size, (rank + 1) * size // world)
    return s, max(s, e)


def _pread_fn(path):
    fd = os.open(path, os.O_RDONLY)
    return fd, os.fstat(fd).st_size, (lambda off, n: os.pread(fd, n, off))


def plan_file(path, rank, world, kind_=None):
    """('sam', split.Share) or ('bam', BamShare) of `rank` for a regular SAM or BAM file; None for an empty one."""
    from .split import Share
    kind_ = kind_ or kind(path)
    fd, size, read = _pread_fn(path)
    try:
        if kind_ is None or size == 0:
            return None
        if kind_ == "sam":
            s, e = plan_sam_share(read, size, rank, world)
            return "sam", Share("sam", s, s, e)
        if kind_ == "bam":
            return "bam", plan_bam_share(read, size, rank, world)
        raise ValueError("%s cannot be split" % kind_)
    finally:
        os.close(fd)


class BamShareReader(object):
    """Rank r's share of a BAM file (BamShare) inflated piece by piece: piece i is the inflated data of a run of whole
    blocks (the first cut at the share's start, the last at its end) of at most `piece_bytes` bytes, or one block when a
    block holds more.  Every block is checked (CRC32, ISIZE).  A share that starts at a record gets EMPTY_BAM_HEADER in
    front, so that the engine reads it from its first record on.  The blocks of a piece are inflated on a pool of
    `threads` threads (zlib releases the GIL), and prefetch(i) inflates piece i on a thread while the caller works on
    piece i - 1.  read(i) -> (bytes, begin, end).  bam=False: the blocks hold SAM text (a bgzip'd SAM file, read whole
    with share = BamShare((0, 0), (size, 0)))."""

    def __init__(self, path, share, piece_bytes, threads=8, bam=True):
        import concurrent.futures
        self.fd, size, read = _pread_fn(path)
        self.share = share
        self.bam = bam
        (b0, o0), (b1, o1) = share.start, share.end
        blocks = walk_blocks(read, size, b0, b1 + (1 if o1 else 0)) if share.start < share.end else []
        self.pieces, cur, n = [], [], 0
        for i, (p, bs, isize) in enumerate(blocks):
            lo = o0 if i == 0 else 0
            hi = o1 if p == b1 else isize
            if cur and n + hi - lo > piece_bytes:
                self.pieces.append(cur)
                cur, n = [], 0
            cur.append((p, bs, lo, hi))
            n += hi - lo
        if cur:
            self.pieces.append(cur)
        self.n_pieces = len(self.pieces)
        self.pool = concurrent.futures.ThreadPoolExecutor(max_workers=max(1, threads))
        self._ahead = None
        self.inflate_s = 0.0              # wall time of reading and inflating the pieces (on the prefetch thread or not)

    def _load(self, i):
        import time
        t0 = time.perf_counter()
        try:
            return self._inflate(i)
        finally:
            self.inflate_s += time.perf_counter() - t0

    def _inflate(self, i):
        blocks = self.pieces[i]
        first, last = blocks[0][0], blocks[-1][0] + blocks[-1][1]
        raw = os.pread(self.fd, last - first, first)
        if len(raw) != last - first:
            raise ValueError("truncated BGZF block at byte %d" % first)

        def one(b):
            p, bs, lo, hi = b
            return inflate_block(raw[p - first:p - first + bs], p)[lo:hi]
        parts = list(self.pool.map(one, blocks))
        if i == 0 and self.share.start != (0, 0):
            parts.insert(0, EMPTY_BAM_HEADER)
        return b"".join(parts), i == 0, i == self.n_pieces - 1

    def prefetch(self, i):
        import threading
        if i >= self.n_pieces or self._ahead is not None:
            return
        box = []

        def run():
            try:
                box.append(self._load(i))
            except BaseException as ex:
                box.append(ex)
        t = threading.Thread(target=run, daemon=True)
        self._ahead = (i, t, box)
        t.start()

    def read(self, i):
        if self._ahead is not None:
            j, t, box = self._ahead
            t.join()
            self._ahead = None
            if j == i:
                if isinstance(box[0], BaseException):
                    raise box[0]
                return box[0]
        return self._load(i)

    def release(self, i):
        pass

    def close(self):
        if self._ahead is not None:
            self._ahead[1].join()
            self._ahead = None
        self.pool.shutdown()
        if self.fd >= 0:
            os.close(self.fd)
            self.fd = -1


class SamShareReader(object):
    """Rank r's lines of a SAM text file (split.Share of format "sam"), read by split's ShareReader into pinned pieces.
    read(i) -> ((pointer, n), begin, end)."""

    bam = False

    def __init__(self, path, share, piece_bytes):
        from .distributed import ShareReader
        self.r = ShareReader(path, share, piece_bytes)
        self.n_pieces = self.r.n_pieces

    def read(self, i):
        hptr, n, begin, end = self.r.read(i)
        return (hptr, n), begin, end

    def prefetch(self, i):
        self.r.prefetch(i)

    def release(self, i):
        self.r.release(i)

    def close(self):
        self.r.close()


def whole_reader(path, owner, piece_bytes):
    """The reader of a whole SAM, gzip'd SAM or BAM file for the rank that owns it (`owner`; the others get no pieces).  A
    regular file in BGZF blocks (BAM, bgzip'd SAM) is inflated block by block on a pool of threads, with host memory
    bounded by two pieces (BamShareReader over the whole file); anything else -- SAM text, other gzip, a pipe -- is read
    whole (WholeSamReader).  CRAM is refused (ValueError)."""
    from .split import splittable
    if owner and splittable(path):
        k = kind(path)
        if k == "cram":
            raise ValueError("CRAM input is not supported ('%s')" % path)
        if k in ("bam", "gz"):
            with open(path, "rb") as f:
                bgzf = block_size(f.read(BGZF_HEAD)) is not None
            if bgzf:
                return BamShareReader(path, BamShare((0, 0), (os.path.getsize(path), 0)), piece_bytes, bam=k == "bam")
    return WholeSamReader(path, owner, piece_bytes)


class WholeSamReader(object):
    """A whole SAM or gzip'd SAM file -- or a pipe -- for the one rank that owns it (`owner`; the others get no pieces):
    read and inflated whole into host memory (gzip with any number of members, streamed), then handed out in pieces of
    `piece_bytes`.  CRAM is refused (ValueError)."""

    def __init__(self, path, owner, piece_bytes):
        import gzip
        import io
        self.data, self.bam = b"", False
        if owner:
            with open(path, "rb") as f:
                raw = f.read()
            if raw.startswith(b"CRAM"):
                raise ValueError("CRAM input is not supported ('%s')" % path)
            if raw[:2] == b"\x1f\x8b":
                # (gzip.decompress copies the rest of the input once per member: quadratic in the members of a BGZF file)
                with gzip.GzipFile(fileobj=io.BytesIO(raw)) as g:
                    raw = g.read()
            self.data = raw
            self.bam = self.data[:4] == b"BAM\1"
        self.piece = max(1, piece_bytes)
        self.n_pieces = (len(self.data) + self.piece - 1) // self.piece

    def read(self, i):
        off = i * self.piece
        return self.data[off:off + self.piece], i == 0, i == self.n_pieces - 1

    def prefetch(self, i):
        pass

    def release(self, i):
        pass

    def close(self):
        self.data = b""
