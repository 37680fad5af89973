"""An exact k-mer counter in plain torch, independent of the engine's kernels, and a digester of binary/sorted dumps.

Both reduce a set of (canonical key, count) pairs to the same per-partition digests, so a count of billions of k-mers can be
compared with a dump of billions of records without holding either.  The code runs on `cuda` and on `cpu` alike.

Keys are the 2k-bit canonical integers of jellyfish_b200.engine (`mer_to_int`, `canonical_int`): A=0 C=1 G=2 T=3, first base
most significant, min(forward, reverse complement).  They are held as int64 words, least significant word first (one word
for k <= 32, two for k <= 64), the layout jfgpu_lookup takes.  torch has no unsigned 64-bit arithmetic: `>>` on int64 is
arithmetic, so every right shift is masked, and unsigned comparisons flip the sign bit first.

A key's partition is the top bits of h(key), a splitmix64 finalizer of its words.  The digest of a partition is
  [number of distinct keys, sum of counts, sum of h(key) mod 2^64, sum of count * h'(key) mod 2^64]
with h' = mix(h ^ SALT), plus the histogram of counts in the bins of HashCounter.histogram(N_BINS) (the last bin collects
every larger count).
"""
import ctypes as C

import torch

N_BINS = 10002
SIGN = -(1 << 63)
SALT = 0x2545F4914F6CDD1D
_M1, _M2 = 0xBF58476D1CE4E5B9, 0x94D049BB133111EB
NL = ord("\n")


def _s64(x):
    """A 64-bit unsigned Python int as the int64 with the same bits."""
    x &= (1 << 64) - 1
    return x - (1 << 64) if x >> 63 else x


def _shr(x, s):
    """Logical right shift of an int64 tensor."""
    return (x >> s) & ((1 << (64 - s)) - 1)


def mix(x):
    """The splitmix64 finalizer of an int64 tensor (products wrap mod 2^64)."""
    x = (x ^ _shr(x, 30)) * _s64(_M1)
    x = (x ^ _shr(x, 27)) * _s64(_M2)
    return x ^ _shr(x, 31)


def key_hash(words):
    """h(key) of keys given as (n, W) int64 words."""
    h = mix(words[:, 0])
    for j in range(1, words.shape[1]):
        h = mix(h ^ words[:, j])
    return h


def partition_of(h, P):
    """The partition of a key with hash h: the top log2(P) bits."""
    bits = P.bit_length() - 1
    return _shr(h, 64 - bits) if bits else torch.zeros_like(h)


def n_words(k):
    assert 1 <= k <= 64, "the model takes k <= 64"
    return 1 if k <= 32 else 2


def _ult(a, b):
    """Unsigned a < b of int64 tensors."""
    return (a ^ SIGN) < (b ^ SIGN)


def _lex_less(a, b, unsigned=False):
    """a < b for (n, W) keys, most significant word last; signed words unless `unsigned`."""
    if unsigned:
        a, b = a ^ SIGN, b ^ SIGN
    lt = a[:, 0] < b[:, 0]
    for j in range(1, a.shape[1]):
        lt = (a[:, j] < b[:, j]) | ((a[:, j] == b[:, j]) & lt)
    return lt


def canonical_words(col, n, k):
    """Canonical keys of n k-mers, (n, W) int64; col(j) gives the codes (int64, shape (n,)) of base j of every k-mer."""
    W = n_words(k)
    dev = col(0).device
    fwd = [torch.zeros(n, dtype=torch.int64, device=dev) for _ in range(W)]
    rc = [torch.zeros(n, dtype=torch.int64, device=dev) for _ in range(W)]
    for j in range(k):
        c = col(j)
        s = 2 * (k - 1 - j)                 # base j of the forward strand: bits s, s+1
        fwd[s >> 6] |= c << (s & 63)
        s = 2 * j                           # its complement is base k-1-j of the reverse complement
        rc[s >> 6] |= (3 - c) << (s & 63)
    fwd, rc = torch.stack(fwd, 1), torch.stack(rc, 1)
    return torch.where(_lex_less(rc, fwd, unsigned=True)[:, None], rc, fwd)


_LUT = {}


def _code_lut(dev):
    if dev not in _LUT:
        lut = torch.full((256,), -1, dtype=torch.int64)
        for i, ch in enumerate(b"ACGT"):
            lut[ch] = i
        _LUT[dev] = lut.to(dev)
    return _LUT[dev]


def codes_of(bytes_u8):
    """ACGT bytes (uint8 tensor) -> codes 0..3 (int64), -1 for any other byte."""
    return _code_lut(bytes_u8.device)[bytes_u8.long()]


def mers_words(mers_u8, k):
    """Canonical keys of k-mers given as an (n, k) uint8 tensor of ACGT bytes."""
    codes = codes_of(mers_u8)
    assert bool((codes >= 0).all()), "a k-mer holds a byte other than ACGT"
    return canonical_words(lambda j: codes[:, j], codes.shape[0], k)


def random_words(n, k, seed, device):
    """n canonical keys of iid random k-mers (seeded)."""
    g = torch.Generator().manual_seed(seed)
    codes = torch.randint(0, 4, (n, k), generator=g, dtype=torch.int64).to(device)
    return canonical_words(lambda j: codes[:, j], n, k)


def sort_words(words):
    """(n, W) keys in ascending signed lexicographic order (most significant word last), by stable sorts."""
    if words.shape[1] == 1:
        return torch.sort(words[:, 0])[0][:, None]
    order = torch.argsort(words[:, 0], stable=True)
    for j in range(1, words.shape[1]):
        order = order[torch.argsort(words[order, j], stable=True)]
    return words[order]


def count_runs(sorted_words):
    """-> (distinct keys (m, W), their counts (m,)) of sorted keys."""
    n = sorted_words.shape[0]
    new = torch.ones(n, dtype=torch.bool, device=sorted_words.device)
    if n > 1:
        new[1:] = (sorted_words[1:] != sorted_words[:-1]).any(1)
    starts = torch.nonzero(new).flatten()
    ends = torch.cat([starts[1:], torch.tensor([n], device=starts.device)])
    return sorted_words[starts], ends - starts


def lower_bound(sorted_words, q):
    """Index of the first key not less than each query (vectorised binary search in the signed order of sort_words)."""
    n = sorted_words.shape[0]
    lo = torch.zeros(q.shape[0], dtype=torch.int64, device=q.device)
    hi = torch.full_like(lo, n)
    for _ in range(max(1, n).bit_length() + 1):
        live = lo < hi
        mid = torch.clamp((lo + hi) // 2, max=max(n - 1, 0))
        less = live & _lex_less(sorted_words[mid], q) if n else torch.zeros_like(live)
        lo = torch.where(less, mid + 1, lo)
        hi = torch.where(live & ~less, mid, hi)
    return lo


def digest_rows(words, counts, P):
    """Per-partition digests of distinct keys with their counts: ((P, 4) int64, (P, N_BINS) int64), on the keys' device."""
    dev = words.device
    h = key_hash(words)
    part = partition_of(h, P)
    dig = torch.zeros((P, 4), dtype=torch.int64, device=dev)
    dig[:, 0] = torch.bincount(part, minlength=P)
    dig[:, 1].index_add_(0, part, counts)
    dig[:, 2].index_add_(0, part, h)
    dig[:, 3].index_add_(0, part, counts * mix(h ^ _s64(SALT)))
    del h
    hist = torch.bincount(part * N_BINS + torch.clamp(counts, max=N_BINS - 1), minlength=P * N_BINS).view(P, N_BINS)
    return dig, hist


class Model(object):
    """What `count` found: n_kmers, P, digest (P, 4) and hist (P, N_BINS) on the CPU, query_counts (CPU int64)."""

    def distinct(self):
        return int(self.digest[:, 0].sum())

    def histogram(self):
        return self.hist.sum(0).tolist()


def choose_partitions(n_kmers, k, device):
    """P (a power of two, at least 8) such that sorting one partition takes under a quarter of the free device memory, and
    how many partitions one pass over the text can gather (every key of a pass is held until its partitions are counted)."""
    kbytes = 8 * n_words(k) * max(n_kmers, 1)
    free = torch.cuda.mem_get_info(device)[0] if torch.device(device).type == "cuda" else 16 << 30
    P = 8
    while 8 * kbytes / P > free / 4 and P < (1 << 16):
        P *= 2
    keep = 0.55 * free - 8 * kbytes / P
    per_pass = max(1, min(P, int(keep / (1.1 * kbytes / P))))
    return P, per_pass


def _fasta_body_start(text):
    head = text[:1 << 16]
    assert int(head[0]) == ord(">"), "not a FASTA record"
    nl = torch.nonzero(head == NL)
    assert len(nl), "no end to the header line"
    return int(nl[0]) + 1


def _chunks(text, k, chunk_bases):
    """Codes (int64) of the sequence of a one-record FASTA text, in pieces that overlap by k - 1 bases."""
    pos = _fasta_body_start(text)
    n = text.numel()
    carry = text.new_zeros(0, dtype=torch.int64)
    while pos < n:
        raw = text[pos:pos + chunk_bases]
        pos += raw.numel()
        codes = codes_of(raw[raw != NL])
        assert bool((codes >= 0).all()), "the sequence holds a byte other than ACGT or a newline"
        codes = torch.cat([carry, codes])
        if codes.numel() >= k:
            yield codes
        carry = codes[max(0, codes.numel() - (k - 1)):]


def _keys(codes, k):
    n = codes.numel() - k + 1
    return canonical_words(lambda j: codes[j:j + n], n, k)


def iter_partitions(text, k, P, parts, chunk_bases):
    """Yield (p, distinct keys, counts) for p in `parts` (consecutive), after one pass over the text.  Also yields the
    number of k-mers of the text as (None, n_kmers, None) first."""
    parts = list(parts)
    pieces = {p: [] for p in parts}
    n_kmers = 0
    for codes in _chunks(text, k, chunk_bases):
        w = _keys(codes, k)
        n_kmers += w.shape[0]
        part = partition_of(key_hash(w), P)
        if len(parts) == P:
            order = torch.argsort(part)
            w, part = w[order], part[order]
            ends = torch.cumsum(torch.bincount(part, minlength=P), 0).tolist()
            for p, (a, b) in enumerate(zip([0] + ends[:-1], ends)):
                pieces[p].append(w[a:b].clone())
        else:
            for p in parts:
                pieces[p].append(w[part == p])
        del w, part
    yield None, n_kmers, None
    for p in parts:
        ks = torch.cat(pieces.pop(p)) if pieces[p] else text.new_zeros((0, n_words(k)), dtype=torch.int64)
        uniq, counts = count_runs(sort_words(ks))
        del ks
        yield p, uniq, counts


def count(text, k, P=None, chunk_bases=None, queries=None, per_pass=None):
    """Count the canonical k-mers of a one-record FASTA text (a uint8 tensor: '>' header line, then ACGT and newlines only).

    P partitions (default: from the free device memory), gathered per_pass at a time, chunks of chunk_bases bytes that
    overlap by k - 1 bases, queries an optional (m, W) int64 tensor of canonical keys whose counts are returned.
    -> Model."""
    dev = text.device
    W = n_words(k)
    if P is None:
        P, fit = choose_partitions(text.numel(), k, dev)
    else:
        fit = P
    per_pass = per_pass or fit
    chunk_bases = chunk_bases or (1 << 27) // W
    digest = torch.zeros((P, 4), dtype=torch.int64, device=dev)
    hist = torch.zeros((P, N_BINS), dtype=torch.int64, device=dev)
    if queries is not None:
        queries = queries.to(dev)
        qpart = partition_of(key_hash(queries), P)
        qcount = torch.zeros(queries.shape[0], dtype=torch.int64, device=dev)
    n_kmers = None
    for p0 in range(0, P, per_pass):
        for p, uniq, counts in iter_partitions(text, k, P, range(p0, min(P, p0 + per_pass)), chunk_bases):
            if p is None:
                n_kmers = uniq
                continue
            d, hst = digest_rows(uniq, counts, P)
            digest += d
            hist += hst
            if queries is not None:
                qi = torch.nonzero(qpart == p).flatten()
                if qi.numel() and uniq.shape[0]:
                    q = queries[qi]
                    at = lower_bound(uniq, q)
                    atc = torch.clamp(at, max=uniq.shape[0] - 1)
                    hit = (at < uniq.shape[0]) & (uniq[atc] == q).all(1)
                    qcount[qi] = torch.where(hit, counts[atc], torch.zeros_like(at))
            del uniq, counts
    m = Model()
    m.k, m.P, m.n_kmers = k, P, n_kmers
    m.digest, m.hist = digest.cpu(), hist.cpu()
    m.query_counts = qcount.cpu() if queries is not None else None
    return m


def partition_counts(text, k, P, p, chunk_bases=None):
    """(distinct keys, counts) of partition p alone: one pass over the text (for a diagnosis)."""
    it = iter_partitions(text, k, P, [p], chunk_bases or (1 << 27) // n_words(k))
    next(it)
    _, uniq, counts = next(it)
    return uniq, counts


def position_tables(k, size, columns, device):
    """(key bytes, 256) int64 tables: the XOR of a key's tables at its little-endian bytes is M * key (the hash matrix with
    these columns, RectangularBinaryMatrix::times as jfutil.positions); modulo size, its original position."""
    c = len(columns)
    assert c == 2 * k, "a matrix of %d columns for k = %d" % (c, k)
    kb = (2 * k + 7) // 8
    tab = [[0] * 256 for _ in range(kb)]
    for b in range(kb):
        for v in range(1, 256):
            low = (v & -v).bit_length() - 1
            i = 8 * b + low
            tab[b][v] = tab[b][v & (v - 1)] ^ (columns[c - 1 - i] if i < c else 0)
    return torch.tensor([[_s64(x) for x in row] for row in tab], dtype=torch.int64, device=device)


class StreamDigest(object):
    """Digests of a binary/sorted body fed in slices (any cut, records may straddle slices): key bytes then ocl count bytes
    per record.  It also checks that (original position, key) strictly increases over the whole stream: a key stored in two
    slots has one original position, so it shows up as two equal records."""

    def __init__(self, k, size, columns, ocl, P, device):
        self.k, self.size, self.ocl, self.P, self.dev = k, size, ocl, P, torch.device(device)
        self.W = n_words(k)
        self.kb = (2 * k + 7) // 8
        self.rec = self.kb + ocl
        self.pos_tab = position_tables(k, size, columns, self.dev)
        self.digest = torch.zeros((P, 4), dtype=torch.int64, device=self.dev)
        self.hist = torch.zeros((P, N_BINS), dtype=torch.int64, device=self.dev)
        self.rest = torch.zeros(0, dtype=torch.uint8, device=self.dev)
        self.last = None                    # (position, key words) of the last record so far
        self.n_records = 0
        self.n_disorder = 0
        self.first_disorder = None          # (record index, its position, the previous record's position)

    def feed_address(self, ptr, n):
        """A slice in host memory, taken without a copy (e.g. the pinned buffer a jfgpu_dump sink receives)."""
        if n:
            self.feed(torch.frombuffer((C.c_uint8 * n).from_address(ptr), dtype=torch.uint8))

    def positions(self, a):
        """Original positions of the records of an (m, rec) uint8 tensor."""
        pos = torch.zeros(a.shape[0], dtype=torch.int64, device=a.device)
        for b in range(self.kb):
            pos ^= self.pos_tab[b][a[:, b].long()]
        return pos & (self.size - 1)

    def words(self, a):
        w = []
        for j in range(self.W):
            x = torch.zeros(a.shape[0], dtype=torch.int64, device=a.device)
            for b in range(8 * j, min(self.kb, 8 * j + 8)):
                x |= a[:, b].long() << (8 * (b - 8 * j))
            w.append(x)
        return torch.stack(w, 1)

    def feed(self, t):
        t = t.to(self.dev)
        if self.rest.numel():
            t = torch.cat([self.rest, t])
        m = t.numel() // self.rec
        self.rest = t[m * self.rec:].clone()
        if not m:
            return
        a = t[:m * self.rec].view(m, self.rec)
        words = self.words(a)
        counts = torch.zeros(m, dtype=torch.int64, device=self.dev)
        for b in range(self.ocl):
            counts |= a[:, self.kb + b].long() << (8 * b)
        pos = self.positions(a)
        if self.last is not None:
            ppos, pw = torch.cat([self.last[0], pos]), torch.cat([self.last[1], words])
        else:
            ppos, pw = pos, words
        ok = (ppos[1:] > ppos[:-1]) | ((ppos[1:] == ppos[:-1]) & _lex_less(pw[:-1], pw[1:], unsigned=True))
        bad = int((~ok).sum())
        if bad and self.first_disorder is None:
            i = int(torch.nonzero(~ok)[0])
            base = self.n_records - (1 if self.last is not None else 0)
            self.first_disorder = (base + i + 1, int(ppos[i + 1]), int(ppos[i]))
        self.n_disorder += bad
        self.last = (pos[-1:].clone(), words[-1:].clone())
        d, h = digest_rows(words, counts, self.P)
        self.digest += d
        self.hist += h
        self.n_records += m

    def finish(self):
        assert self.rest.numel() == 0, "the stream ends inside a record (%d bytes left)" % self.rest.numel()
        self.digest, self.hist = self.digest.cpu(), self.hist.cpu()
        return self


def differing_partitions(model, digest):
    """Partitions whose digest or histogram differ between a Model and a finished StreamDigest (or two Models)."""
    bad = (model.digest != digest.digest).any(1) | (model.hist != digest.hist).any(1)
    return torch.nonzero(bad).flatten().tolist()
