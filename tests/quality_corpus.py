"""4-line FASTQ texts that aim the events of the -Q quality filter at the ends of staging batches.

A batch of B bytes is cut into tiles of TILE bytes; its last tile holds r = B - (ceil(B / TILE) - 1) * TILE bytes, and the
last window of K1 starts at h = E - r - HALO, where E is the batch end (seam_corpus.py names the constants).  K1 hands the
next batch a carry of the last PRE (PRE_WIDE for k > 64) symbols of the text.  When that window starts in a sequence line,
emits no reset in its halo and fewer symbols than the carry holds, the carry is rebuilt from the bytes in front of E, and
the next batch builds its first k-mers from it (jf_extract.cuh, the carry hand-over).

One cell sits at every batch end.  Laid out backwards from E:

  S1      a sequence line whose '\\n' is at h + a (a = bytes of S1 inside the window), good qualities;
  +, Q1   its '+' line and its quality line, which run on through the halo;
  H2      the next header, "@" + name, ending right in front of S2 (so it starts in the tile when S2 starts late);
  S2      the next sequence line, from s2 = E + s2_off on, at least k + 6 bases past E, with low-quality bases at the
          given offsets from E (a negative offset is a byte in front of E).

Filler records fill the bytes between cells; their qualities are all '!' (below any threshold used here), so under -Q
they add resets only.  `cell_texts` also returns where every part of every cell landed, which
tests/test_quality_corpus_cpu.py checks against the bytes."""
import random

import numpy as np

import seam_corpus as sc

HALO, PRE, PRE_WIDE = sc.HALO, sc.PRE, sc.PRE_WIDE
GOOD = ord("I")
FILL_Q = ord("!")
FILL_MAX = 3000                     # read length of the filler records


def last_tile(batch, tile):
    """Length of the last tile of a batch of `batch` bytes (0 < r <= tile)."""
    return batch - (-(-batch // tile) - 1) * tile


def prek(k):
    """Symbols the carry holds for k."""
    return PRE_WIDE if k > 64 else PRE


def record(name, seq, qual, eol=b"\n"):
    return b"@" + name + eol + seq + eol + b"+" + eol + qual + eol


def filler(n, rng, eol=b"\n"):
    """Exactly n bytes of 4-line records whose qualities are all '!' (n >= 6 + 4 len(eol))."""
    e = len(eol)
    out = []
    while n:
        full = 2 * FILL_MAX + 2 + 4 * e + 1
        if n >= full + 2 * FILL_MAX:
            name, ln = b"f", FILL_MAX
        else:
            nl = 1 + (n - 2 - 4 * e - 1) % 2                 # the name takes the odd byte
            ln = (n - 2 - 4 * e - nl) // 2
            assert ln >= 1, n
            name = b"f" * nl
        out.append(record(name, sc.bases(ln, rng), bytes([FILL_Q]) * ln, eol))
        n -= len(out[-1])
    return b"".join(out)


def cell(s2_off, low=(), lowq=ord("#"), a=2, eol=b"\n", name=b"GATTACA"):
    """One batch-end cell (see the module docstring).  `name` ends the header of S2 (bases: a carry that walked back into
    the header would pick them up)."""
    return {"s2_off": s2_off, "low": tuple(low), "lowq": lowq, "a": a, "eol": eol, "name": name}


def _lay_cell(E, h, c, k, i, rng):
    """-> (first byte, bytes, placement) of the two records of cell c at batch end E."""
    eol, e = c["eol"], len(c["eol"])
    s2 = E + c["s2_off"]
    l2 = E + k + 6 - s2
    q2 = bytearray([GOOD]) * l2
    for o in c["low"]:
        j = E + o - s2
        assert 0 <= j < l2, (o, c)
        q2[j] = c["lowq"]
    h2 = b"@q%d" % i + c["name"] + eol
    hs = s2 - len(h2)
    nl1 = h + c["a"]                                         # the '\n' of S1
    s1_body = hs - nl1 - 2 - 2 * e                           # Q1 runs from nl1 + 2 + e to the header, as long as S1
    assert s1_body >= c["a"] + 1, (s1_body, c)               # (with DOS ends S1's last byte, '\r', is inside it)
    h1 = b"@p%d" % i + eol
    s1 = nl1 - (e - 1) - s1_body
    first = s1 - len(h1)
    out = h1 + sc.bases(s1_body, rng) + eol + b"+" + eol + bytes([GOOD]) * s1_body + eol
    assert first + len(out) == hs
    out += h2 + sc.bases(l2, rng) + eol + b"+" + eol + bytes(q2) + eol
    q2_start = s2 + l2 + e + 1 + e
    place = dict(c, E=E, h=h, s1=s1, nl1=nl1, hs=hs, s2=s2, l2=l2, q2=q2_start, end=first + len(out))
    return first, out, place


def aimed_cells(k, min_qual, full=True):
    """The cells of one sweep: the low-quality base at every offset of the carry in front of E (S2 starting one byte before
    it), S2 starting at every offset in [E - PRE - 2, E + 2] (a low-quality base halfway between s2 and E), quality bytes
    at the threshold, one below it and >= 0x80, DOS line ends, and several low-quality bases.  full=False: the ends and
    the middle of the two sweeps only."""
    pk = prek(k)
    lows = range(1, pk + 1) if full else sorted({1, 2, 3, k - 3, k - 2, k - 1, k, k + 1, pk - 2, pk - 1, pk} & set(range(1, pk + 1)))
    starts = range(-pk - 2, 3) if full else sorted({-pk - 2, -pk - 1, -pk, -pk + 1, -k - 1, -k, -k + 1, -3, -2, -1, 0, 1, 2})
    cells = [cell(-(o + 1), low=[-o]) for o in lows]
    cells += [cell(d, low=[d // 2] if d <= -2 else []) for d in starts]
    cells += [cell(-20, low=[-5], lowq=q) for q in (min_qual, min_qual - 1, 0x80, 0xF0)]
    cells += [cell(-20, low=[-5], eol=b"\r\n", a=a) for a in (0, 3)] + [cell(1, eol=b"\r\n", a=0), cell(-9, eol=b"\r\n", a=0)]
    cells += [cell(-40, low=[-3, -9, -30]), cell(2, name=b"7"), cell(-5, low=[-2], a=0)]
    return cells


def cell_texts(batch, tile, k, cells, seed=1, per_text=None):
    """Texts with cells[i] at the end of batch i (of `batch` bytes) -> list of (text, [placement]).  A placement is the
    cell with where it landed: E, h, s1 (first base of S1), nl1, hs (header of S2), s2, l2 (bases of S2), q2 (first
    quality byte of S2), end (first byte after the cell)."""
    rng = random.Random(seed)
    r = last_tile(batch, tile)
    texts = []
    per_text = per_text or len(cells)
    for t0 in range(0, len(cells), per_text):
        out, at, placed = [], 0, []
        for j, c in enumerate(cells[t0:t0 + per_text]):
            E = (j + 1) * batch
            first, body, place = _lay_cell(E, E - r - HALO, c, k, t0 + j, rng)
            gap = first - at
            assert gap >= 10 or gap == 0, (gap, c)
            out.append(filler(gap, rng))
            out.append(body)
            placed.append(place)
            at = first + len(body)
        out.append(filler(2 * batch // 3 + 17, rng))          # the text ends inside one more batch
        texts.append((b"".join(out), placed))
    return texts


def window_symbols(p, min_qual):
    """What the generator claims of the last window of the batch that ends at p["E"]: (symbols it emits, whether it emits
    a reset in its halo), counted from the layout (S1's tail, S2's header reset, S2 up to E) under -Q `min_qual` (0: the
    default parser)."""
    E, h = p["E"], p["h"]
    cr = len(p["eol"]) == 2 and p["a"] > 0                   # S1's '\r' is inside the window
    n = p["a"] - (cr and not min_qual)                        # (the default parser drops a line-end '\r'; -Q keeps it)
    halo_reset = bool(min_qual) and cr
    if p["hs"] < E:
        n += 1                                               # the header's reset
        halo_reset |= p["hs"] < h + HALO
    n += max(0, E - p["s2"])
    if min_qual and p["lowq"] < min_qual:
        halo_reset |= any(E + o < h + HALO for o in p["low"])
    return n, halo_reset


def carry_is_rebuilt(p, k, min_qual, batch, tile):
    """Whether the batch that ends at p["E"] hands over a carry rebuilt from its bytes (the backfill): its last tile is not
    its first one, its last window starts in a sequence line (S1), emits no reset in its halo and fewer symbols than the
    carry holds."""
    n, halo_reset = window_symbols(p, min_qual)
    return batch > tile and p["s1"] <= p["h"] <= p["nl1"] and not halo_reset and n < prek(k)


def one_cell_text(E, tile, k, c, n_bytes, seed=1):
    """A text of n_bytes (> E) with cell c at byte E, the end of a batch of E bytes, built as a numpy array: filler records
    of 3000 bases in front, and behind.  -> (text, the bytes of the cell's two records, placement).  Under -Q the filler
    adds resets only, so the k-mers of the cell's records alone are those of the whole text."""
    rng = random.Random(seed)
    first, body, place = _lay_cell(E, E - last_tile(E, tile) - HALO, c, k, 0, rng)
    rec = np.frombuffer(record(b"f", b"A" * FILL_MAX, bytes([FILL_Q]) * FILL_MAX), np.uint8)
    text = np.empty(n_bytes, np.uint8)
    reps = max(0, (first - 3 * len(rec)) // len(rec))
    text[:reps * len(rec)] = np.tile(rec, reps)
    head = filler(first - reps * len(rec), rng)
    text[reps * len(rec):first] = np.frombuffer(head, np.uint8)
    text[first:first + len(body)] = np.frombuffer(body, np.uint8)
    at = first + len(body)
    reps = max(0, (n_bytes - at - 3 * len(rec)) // len(rec))
    text[at:at + reps * len(rec)] = np.tile(rec, reps)
    at += reps * len(rec)
    text[at:] = np.frombuffer(filler(n_bytes - at, rng), np.uint8)
    return text, body, place
