"""Deterministic texts that put every parser event of the extraction pipeline (K0a nl_scan, K0b tile_state, K1 extract)
right at the places where its state is cut: window and tile boundaries, staging-batch ends and feed-call cuts.

The constants below are the ones the pipeline uses; a test that relies on a seam falling at a given byte names it here.
"""
import random

import numpy as np

HALO = 256                      # jellyfish_b200/csrc/jf_device.cuh:21  bytes of the previous tile in front of a window
PRE = 64                        # jf_device.cuh:22  symbols a Carry holds for k <= 64
PRE_WIDE = 128                  # jf_device.cuh:23  the same for k > 64
TILE_512 = 512 * 32 - HALO      # jf_engine.cu:965 (run_batch)  tile of the 512-thread K1 (direct insert, route, query) = 16128
TILE_1024 = 1024 * 32 - HALO    # jf_engine.cu:965 (run_batch)  tile of the 1024-thread K1 (region records, record exchange) = 32512
TILES = (TILE_512, TILE_1024)
DENSE_PERIOD = 1009             # prime: coprime to every tile, split and batch length used here


def batch_len(max_batch_bytes):
    """The staging batch the engine uses for a max_batch_bytes: rounded up to 16 bytes (jf_engine.cu:1484, jfgpu_create)."""
    return (max_batch_bytes + 15) & ~15


def bases(n, rng):
    return bytes(rng.choice(b"ACGT") for _ in range(n)) if n < 64 else \
        np.frombuffer(b"ACGT", np.uint8)[np.random.default_rng(rng.getrandbits(32)).integers(0, 4, n)].tobytes()


def fasta_events(k, batch):
    """name -> bytes of every FASTA event; each is inserted into the middle of a sequence line."""
    rng = random.Random(5)
    one_per_line = b"".join(bytes([c]) + b"\r\n" for c in bases(k + 2, rng))
    ev = {
        "header": b"\n>seam header\n",
        "long_header": b"\n>" + b"H" * 70000 + b"\n",
        "header_cr": b"\n>a\rb\r\n",
        "two_headers": b"\n>a\n>b\n",
        "header_only": b"\n>only a header\n>next\n",
        "lone_nl": b"\n",
        "blank_run": b"\n" * 300,
        "one_per_line": b"\n" + one_per_line,
        "cr_nl": b"\r\n",
        "cr_run_nl": b"\r\r\r\n",
        "cr_base": b"\r",
        "cr_line_start": b"\n\r\r",
        "cr_255": b"\r" * 255,
        "cr_256": b"\r" * 256,
        "cr_257": b"\r" * 257,
        "N": b"N", "n": b"n", "iupac": b"RYKMSWBDHV", "dash": b"-", "space": b" ", "gt_mid": b">",
        "x_c1": b"\xc1", "x_e1": b"\xe1", "x_e7": b"\xe7", "ctrl": b"\x00\x01\x7f\t",
    }
    if batch:
        ev["cr_batch"] = b"\r" * batch
        ev["cr_batch_1"] = b"\r" * (batch - 1)
    return ev


def _background(n, rng, width=61):
    """n bytes of sequence lines (a '\\n' every `width` bytes)."""
    s = bytearray(bases(n, rng))
    s[width - 1::width] = b"\n" * len(s[width - 1::width])
    return bytes(s)


def _lay_out(targets, rng, head=b">seam corpus\n"):
    """A FASTA text with events[i] starting at byte targets[i][0] (targets sorted, events that would overlap are dropped)
    -> (text, [(position, label)])."""
    out = [head]
    at = len(head)
    placed = []
    for pos, label, ev in targets:
        if pos < at:
            continue
        out.append(_background(pos - at, rng))
        out.append(ev)
        placed.append((pos, label))
        at = pos + len(ev)
    out.append(_background(2000, rng) + b"\n")
    return b"".join(out), placed


def seams(tile, n_bytes, batch=0):
    """(position, name) of every seam of a text of n_bytes fed as batches of `batch` bytes (0: one batch): the tile starts
    and the TILE - HALO splits of K0a, counted from every batch start, and the batch ends."""
    out = []
    starts = range(0, n_bytes, batch) if batch else [0]
    for b0 in starts:
        b1 = min(n_bytes, b0 + batch) if batch else n_bytes
        for t0 in range(b0, b1, tile):
            if t0 > b0:
                out.append((t0, "tile"))
            out.append((t0 + tile - HALO, "split"))
        if batch and b1 < n_bytes:
            out.append((b1, "batch"))
    return sorted(set(out))


def seam_texts(k, tile, events, batch=0, max_bytes=3 << 20, seed=1, offs=None):
    """Texts that place every event at every offset d in `offs` (default [-(k+2), k+2]) of a window start ("tile") and of
    a K0a split ("split"): each kind of seam takes the (event, offset) pairs in turn with a cursor of its own, until both
    kinds have had every pair.  Batch ends ("batch") take the pairs in turn too, as many as the texts hold (a batch end
    comes once every batch / tile windows).  -> list of (text, [(position, label)]) with label "event@seam%+d"."""
    names = sorted(events)
    offs = list(range(-(k + 2), k + 3)) if offs is None else list(offs)
    combos = [(names[i % len(names)], offs[(i // len(names)) % len(offs)]) for i in range(len(names) * len(offs))]
    rng = random.Random(seed)
    texts = []
    cur = {"tile": 0, "split": 0, "batch": 0}
    while min(cur["tile"], cur["split"]) < len(combos):
        targets = []
        free = 1024                                   # first byte the next event may take
        for pos, kind in seams(tile, max_bytes, batch):
            if pos > max_bytes - 80000:
                break
            if kind != "batch" and cur[kind] >= len(combos):
                continue
            name, d = combos[cur[kind] % len(combos)]
            if pos + d < free:
                continue                              # (a long event covers this seam: the pair goes to the next one)
            targets.append((pos + d, "%s@%s%+d" % (name, kind, d), events[name]))
            free = pos + d + len(events[name]) + 1
            cur[kind] += 1
        texts.append(_lay_out(targets, rng))
    return texts


def dense_text(events, n_bytes, seed=2, period=DENSE_PERIOD):
    """One text with an event every `period` bytes, cycling through the events.  The period is coprime to every tile,
    split and batch length, so the events' positions relative to the seams keep moving: a text of n bytes puts about
    n / period events at distinct residues of each seam (it does not hit every residue)."""
    rng = random.Random(seed)
    names = sorted(n for n in events if len(events[n]) < period // 2)
    targets = [(p, "%s@%d" % (names[i % len(names)], p), events[names[i % len(names)]])
               for i, p in enumerate(range(period, n_bytes, period))]
    return _lay_out(targets, rng)


def fastq_text(n_bytes, k, seed=3, eol=b"\n", quals=b"FGHIJ", low=b"", long_every=0):
    """4-line FASTQ: read lengths 1, k-1, k, k+1 and random ones (and 40 KB every `long_every` reads), quality lines that
    start with '@', '+' or '>', 'N' in reads; `low`: quality bytes placed at random (below a -Q threshold).  Nothing is
    aimed at a seam here: the record boundaries, quality lines and low-quality bases fall at seeded random offsets, so
    the FASTQ coverage of the seams is statistical (a 3 MB text puts over ten thousand record boundaries across its
    ~190 windows)."""
    rng = random.Random(seed)
    out, at, i = [], 0, 0
    while at < n_bytes:
        if long_every and i % long_every == long_every - 1:
            ln = 40000
        else:
            ln = max(1, rng.choice((1, k - 1, k, k + 1, rng.randrange(2, 300), rng.randrange(2, 300))))
        sq = bytearray(bases(ln, rng))
        if rng.random() < 0.2:
            sq[rng.randrange(ln)] = ord(rng.choice("NnR"))
        q = bytearray(rng.choice(quals) for _ in range(ln))
        if i % 7 < 3:
            q[0] = b"@+>"[i % 7]
        for _ in range(rng.randrange(0, 3) if low else 0):
            q[rng.randrange(ln)] = rng.choice(low)
        rec = b"@r%d" % i + eol + bytes(sq) + eol + (b"+" if i % 2 else b"+r%d" % i) + eol + bytes(q) + eol
        out.append(rec)
        at += len(rec)
        i += 1
    return b"".join(out)


def hostile_fasta(n_bytes, rng, events):
    """Random FASTA text of n_bytes built from the event vocabulary (events shorter than 2 KB) and sequence lines of
    random widths, with DOS line ends here and there."""
    names = sorted(n for n in events if len(events[n]) < 2048)
    out = [b">h\n"]
    at = 3
    while at < n_bytes:
        r = rng.random()
        if r < 0.5:
            piece = bases(rng.randrange(1, 200), rng)
        elif r < 0.6:
            piece = rng.choice((b"\n", b"\r\n", b"\r\r\n"))
        else:
            piece = events[rng.choice(names)]
        out.append(piece)
        at += len(piece)
    if rng.random() < 0.5:
        out.append(b"\n")
    return b"".join(out)


def split_points(text, cuts):
    """Feed-call cut points near `cuts` that keep the '\\r' contract of jfgpu_feed: a call ends inside a run of '\\r' only
    when a '\\n' ends the run (the engine takes the end of a call for a line end), so a cut inside a run moves to just
    before its '\\n', or to the run's start when something else follows it; cuts stay increasing."""
    out = []
    for c in sorted(cuts):
        c = min(max(c, 1), len(text) - 1)
        if text[c - 1] == 13:
            r = c
            while r < len(text) and text[r] == 13:
                r += 1
            if r < len(text) and text[r] == 10:
                c = r
            else:
                while c > 1 and text[c - 1] == 13:
                    c -= 1
        if (not out or c > out[-1]) and 0 < c < len(text):
            out.append(c)
    return out
