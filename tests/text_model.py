"""A plain numpy model of the text contract: which k-mers a FASTA / FASTQ text holds, in input order.

It restates `count_file` and `count_file_qual` of oracle/jf_oracle.c (the default parser and the -Q / --min-quality
parser of the reference, DESIGN.md section 7a) line by line, with no per-byte Python loop:

  FASTA    a line whose first byte other than '\\r' is '>' is a header (one reset); blank lines and lines of '\\r' only
           are skipped without a reset; on a sequence line the leading '\\r' run and the trailing '\\r' run are dropped,
           every other byte is a base (ACGTacgt) or a reset -- a '\\r' in the middle of a line, 'N', IUPAC codes, bytes
           >= 0x80 whose low bits spell a base (0xC1, 0xE7), ...
  FASTQ    the header line is dropped, the sequence lines up to the line that starts with '+' are read as FASTA
           sequence lines, the qualities are skipped by length, every read starts with a reset
  -Q       whole_sequence_parser: lines are read with getline, so '\\r' is an ordinary (resetting) byte; a FASTA line
           that starts with '>' opens a record, every other line is sequence; a FASTQ base counts only if its quality
           byte, compared as a signed char, is >= the threshold; every record starts with a reset.  FASTA under -Q
           passes every base.
  files    no k-mer spans two files

`symbols` gives, per file, the stream of base codes 0..3 with BREAK (4) at every reset.  That stream does not depend on
k; `kmers` and `counts` derive the k-mers (1, 2 or 4 little-endian uint64 words, k <= 128) and their exact counts."""
import numpy as np

BREAK = 4
_LUT = np.full(256, BREAK, np.uint8)
for _i, _c in enumerate(b"ACGT"):
    _LUT[_c] = _i
    _LUT[_c | 0x20] = _i
_NL, _CR = 10, 13


def _lines(d):
    """-> (line starts, line ends) of d; a line ends at its '\\n' (exclusive) or at the end of the data."""
    nl = np.flatnonzero(d == _NL)
    return np.concatenate(([0], nl + 1)), np.concatenate((nl, [len(d)]))


def _gather(d, starts, ends):
    """The bytes d[starts[i]:ends[i]] of every range, concatenated, and where each range begins in the result."""
    lens = (ends - starts).astype(np.int64)
    first = np.concatenate(([0], np.cumsum(lens)[:-1])).astype(np.int64)
    total = int(lens.sum())
    rel = np.arange(total, dtype=np.int64) - np.repeat(first, lens)
    return d[np.repeat(starts.astype(np.int64), lens) + rel], first


def _with_breaks(sym, at):
    """sym with a BREAK inserted in front of the positions `at` (sorted)."""
    return np.insert(sym, np.asarray(at, np.int64), BREAK)


def _fasta(d):
    n = len(d)
    ls, le = _lines(d)
    pos = np.arange(n + 1, dtype=np.int64)
    notcr = np.concatenate((d != _CR, [True]))
    nxt = np.minimum.accumulate(np.where(notcr, pos, n)[::-1])[::-1]       # first byte >= i that is not '\r'
    prv = np.maximum.accumulate(np.where(notcr, pos, -1))                  # last byte <= i that is not '\r'
    dx = np.concatenate((d, [_NL]))
    fnc = nxt[ls]
    nonblank = fnc < le
    header = nonblank & (dx[fnc] == ord(">"))
    seq = nonblank & ~header
    s, e = fnc[seq], prv[le[seq] - 1] + 1                                 # leading and trailing '\r' runs dropped
    mark = np.zeros(n + 1, np.int8)
    mark[s] += 1
    mark[e] -= 1
    kept = np.cumsum(mark[:n]) > 0
    sym = np.full(n, 255, np.uint8)
    sym[kept] = _LUT[d[kept]]
    sym[fnc[header]] = BREAK
    return sym[sym != 255]


def _fastq(d):
    """read_fastq + skip_quals of the default parser, restated with bytes.find (one step per line)."""
    b = d.tobytes()
    n = len(b)
    starts, ends, reads = [], [], []
    out_len = 0
    p = b.find(b"\n") + 1 if b.find(b"\n") >= 0 else n                    # first header
    while True:
        seq_len = 0
        while True:                                                         # sequence lines
            while p < n and b[p] in (_NL, _CR):
                p += 1
            if p >= n or b[p] == ord("+"):
                break
            e = b.find(b"\n", p)
            e = n if e < 0 else e
            t = e
            while t > p and b[t - 1] == _CR:
                t -= 1
            starts.append(p)
            ends.append(t)
            out_len += t - p
            seq_len += t - p
            p = e
        if p >= n:
            break
        e = b.find(b"\n", p)                                                # the '+' line
        p = n if e < 0 else e + 1
        quals = 0
        while p < n and quals < seq_len:                                    # qualities, by length
            while p < n and b[p] in (_NL, _CR):
                p += 1
            e = b.find(b"\n", p)
            e = n if e < 0 else e
            e = min(e, p + seq_len - quals)
            t = e
            if e < n and b[e] == _NL:
                while t > p and b[t - 1] == _CR:
                    t -= 1
            quals += t - p
            p = e
        while p < n and b[p] in (_NL, _CR):
            p += 1
        if p >= n:
            break
        if quals != seq_len or b[p] != ord("@"):
            raise ValueError("Invalid fastq sequence")
        reads.append(out_len)
        e = b.find(b"\n", p)                                                # next header
        p = n if e < 0 else e + 1
    raw, _ = _gather(d, np.array(starts, np.int64), np.array(ends, np.int64))
    return _with_breaks(_LUT[raw], reads)


def _fasta_qual(d):
    ls, le = _lines(d)
    keep = ls < le
    ls, le = ls[keep], le[keep]
    header = d[ls] == ord(">")
    raw, first = _gather(d, ls[~header], le[~header])
    # a header's reset goes in front of the first sequence byte that follows it
    after = np.searchsorted(ls[~header], ls[header])
    at = np.concatenate((first, [len(raw)]))[after]
    return _with_breaks(_LUT[raw], at)


def _fastq_qual(d, min_qual):
    b = d.tobytes()
    n = len(b)

    def getline(p):
        e = b.find(b"\n", p)
        return (p, n, n) if e < 0 else (p, e, e + 1)

    ss, se, qs, qe, recs = [], [], [], [], []
    total = 0
    p = 0
    while p < n:
        ns = nq = 0
        p += 1                                                             # '@'
        _, _, p = getline(p)                                               # header
        recs.append(total)
        while p < n and b[p] != ord("+"):
            lb, lend, p = getline(p)
            ss.append(lb), se.append(lend)
            ns += lend - lb
        if p >= n:
            raise ValueError("Truncated fastq file")
        _, _, p = getline(p)                                               # the '+' line
        if ns == 0 and p < n and b[p] != ord("+"):
            lb, lend, p = getline(p)
            qs.append(lb), qe.append(lend)
            nq = lend - lb
        while nq < ns and p < n:
            lb, lend, p = getline(p)
            qs.append(lb), qe.append(lend)
            nq += lend - lb
        if nq != ns:
            raise ValueError("Invalid fastq file: wrong number of quals")
        if p < n and b[p] != ord("@"):
            raise ValueError("Invalid fastq file: header missing")
        total += ns
    seq, _ = _gather(d, np.array(ss, np.int64), np.array(se, np.int64))
    qual, _ = _gather(d, np.array(qs, np.int64), np.array(qe, np.int64))
    sym = _LUT[seq]
    sym[qual.view(np.int8) < np.int8(min_qual)] = BREAK
    return _with_breaks(sym, recs)


def symbols(data, min_qual=0):
    """Base codes 0..3 of one file in input order, BREAK at every reset (the stream starts and ends with one).  min_qual:
    the -Q threshold as a byte value (0: the default parser)."""
    d = np.frombuffer(bytes(data), np.uint8)
    if len(d) == 0:
        return np.array([BREAK], np.uint8)
    if d[0] not in (ord(">"), ord("@")):
        raise ValueError("Unsupported format")
    if min_qual:
        sym = _fasta_qual(d) if d[0] == ord(">") else _fastq_qual(d, min_qual)
    else:
        sym = _fasta(d) if d[0] == ord(">") else _fastq(d)
    return np.concatenate(([BREAK], sym, [BREAK])).astype(np.uint8)


def stream(files, min_qual=0):
    """The symbol streams of several files, one after the other: no k-mer spans two files."""
    return np.concatenate([symbols(f, min_qual) for f in files]) if files else np.array([BREAK], np.uint8)


def _pack(c, L):
    """v[j] = the L codes ending at j packed two bits each, the oldest most significant (valid for j >= L - 1)."""
    v = np.zeros(len(c), np.uint64)
    for i in range(L if len(c) >= L else 0):
        v[L - 1:] |= c[i:len(c) - L + 1 + i] << np.uint64(2 * (L - 1 - i))
    return v


def _words(c, ends, k):
    """The k-mers of codes c ending at `ends`, as (n, nw) little-endian uint64 words."""
    nw = 1 if k <= 32 else 2 if k <= 64 else 4
    out = np.zeros((len(ends), nw), np.uint64)
    full = _pack(c, 32) if k >= 32 else None
    for w in range((k + 31) // 32):
        L = min(32, k - 32 * w)
        out[:, w] = (full if L == 32 else _pack(c, L))[ends - 32 * w]
    return out


def less(a, b):
    """Row-wise a < b of two (n, nw) word arrays (most significant word last)."""
    res = np.zeros(len(a), bool)
    done = np.zeros(len(a), bool)
    for w in range(a.shape[1] - 1, -1, -1):
        ne = ~done & (a[:, w] != b[:, w])
        res[ne] = a[ne, w] < b[ne, w]
        done |= ne
    return res


def kmers(sym, k, canonical=False):
    """Every k-mer of a symbol stream in input order, (n, nw) uint64 words (canonical: the smaller of the k-mer and its
    reverse complement)."""
    n = len(sym)
    pos = np.arange(n, dtype=np.int64)
    last_break = np.maximum.accumulate(np.where(sym == BREAK, pos, -1))
    ends = np.flatnonzero(pos - last_break >= k)
    c = np.where(sym == BREAK, 0, sym).astype(np.uint64)
    fw = _words(c, ends, k)
    if not canonical:
        return fw
    rc = _words((np.uint64(3) - c)[::-1].copy(), n - 1 - (ends - k + 1), k)
    return np.where(less(rc, fw)[:, None], rc, fw)


def _group(w):
    """Rows of an (n, nw) word array grouped by value -> (group of every row, the distinct rows in ascending order, the
    size of every group)."""
    order = np.lexsort(w.T)                       # (the last word, the most significant one, is the primary key)
    s = w[order]
    new = np.ones(len(s), bool)
    new[1:] = np.any(s[1:] != s[:-1], axis=1)
    gs = np.cumsum(new) - 1
    gid = np.empty(len(s), np.int64)
    gid[order] = gs
    return gid, s[new], np.bincount(gs)


def counts(sym, k, canonical=False):
    """-> (unique keys as (m, nw) words in ascending order, their multiplicities, the number of k-mers)."""
    w = kmers(sym, k, canonical)
    if len(w) == 0:
        return w, np.zeros(0, np.int64), 0
    _, keys, cnt = _group(w)
    return keys, cnt, len(w)


def as_ints(words):
    """(n, nw) words -> Python ints."""
    return [sum(int(x) << (64 * i) for i, x in enumerate(row)) for row in words]


def records_to_words(body, k, counter_len):
    """A binary/sorted record body -> ((n, nw) key words, counts), sorted by key like `counts`."""
    nw = 1 if k <= 32 else 2 if k <= 64 else 4
    kb = (2 * k + 7) // 8
    rec = kb + counter_len
    r = np.frombuffer(body, np.uint8).reshape(-1, rec)
    kbuf = np.zeros((len(r), 8 * nw), np.uint8)
    kbuf[:, :kb] = r[:, :kb]
    cbuf = np.zeros((len(r), 8), np.uint8)
    cbuf[:, :counter_len] = r[:, kb:]
    keys = kbuf.view("<u8").reshape(-1, nw)
    cnt = cbuf.view("<u8").reshape(-1).astype(np.int64)
    if len(keys):
        order = np.lexsort(keys.T)
        keys, cnt = keys[order], cnt[order]
    return keys, cnt


def query_lines(sym, k, canonical, keys, cnt):
    """The bytes `query -s` prints for the k-mers of `sym` against a table holding (keys, cnt): "MER COUNT\\n" per k-mer
    in input order (the canonical form when the table is canonical; 0 for an absent k-mer)."""
    w = kmers(sym, k, canonical)
    m = len(w)
    if m == 0:
        return b""
    inv, _, _ = _group(np.concatenate((keys, w)))
    table = np.zeros(int(inv.max()) + 1, np.int64)
    table[inv[:len(keys)]] = cnt
    c = table[inv[len(keys):]]
    nd = np.ones(m, np.int64)
    for p in range(1, 20):
        nd += c >= 10 ** p
    ll = k + 2 + nd
    off = np.concatenate(([0], np.cumsum(ll)[:-1]))
    out = np.empty(int(ll.sum()), np.uint8)
    j = np.arange(k)
    shift = (2 * ((k - 1 - j) % 32)).astype(np.uint64)
    codes = (w[:, (k - 1 - j) // 32] >> shift[None, :]) & np.uint64(3)
    out[off[:, None] + j[None, :]] = np.frombuffer(b"ACGT", np.uint8)[codes.astype(np.int64)]
    out[off + k] = ord(" ")
    for dgt in range(int(nd.max())):
        has = nd > dgt
        p10 = 10 ** (nd[has] - 1 - dgt)
        out[off[has] + k + 1 + dgt] = ord("0") + (c[has] // p10) % 10
    out[off + k + 1 + nd] = ord("\n")
    return out.tobytes()
