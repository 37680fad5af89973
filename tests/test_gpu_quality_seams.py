"""The quality filter (-Q, jfgpu_params.min_qual) against the text model (tests/text_model.py: symbols(text, min_qual), the
restatement of the oracle's count_file_qual) on every K1 insertion path, with its events aimed at the ends of staging
batches (tests/quality_corpus.py).

A device feed cuts its text into batches of a fixed length, so a read runs on across the end of a batch.  The texts here
put, at every batch end, a window that starts at the end of one read's sequence line and the start of the next read's
sequence line in its last tile, with low-quality bases in the symbols the next batch takes over.  The batch length is
j * TILE + r with last tiles r of 16, 96, 256, TILE - 16 and TILE bytes (64 MB and 512 MB both leave r = 256), so the
batch-end geometry of a full-size count is there at a few tens of KB.  The same cells go through the default parser too
(no -Q): there the header in front of the next read ends in bases, which must not reach the next batch either.

Every count case compares the exact (key, count) dump and the statistics with the model and names the first k-mer, in
input order, whose count differs."""
import functools

import numpy as np
import pytest

import quality_corpus as qc
import seam_corpus as sc
import text_model as tm

pytestmark = pytest.mark.gpu

Q = ord("5")
LAST_TILES = ("16", "96", "256", "tile-16", "tile")


@pytest.fixture(scope="module")
def cuda(built):
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    torch.cuda.set_device(0)
    return torch


def _device(torch, data):
    if isinstance(data, np.ndarray):
        t = torch.zeros(len(data) + 16, dtype=torch.uint8, device="cuda")
        t[:len(data)] = torch.from_numpy(data).cuda()
        return t
    t = torch.zeros(len(data) + 16, dtype=torch.uint8, device="cuda")
    if data:
        t[:len(data)] = torch.frombuffer(bytearray(data), dtype=torch.uint8).cuda()
    return t


def _first_diff(text, k, canonical, min_qual, model, got):
    """Index (in input order) and line of the first k-mer of the text (or list of files), every base read as passing, whose count in `got`
    differs from the model's; else the first key the engine holds that no such k-mer has."""
    from jellyfish_b200 import int_to_mer
    sym = tm.stream(text if isinstance(text, list) else [text], -128 if min_qual else 0)   # (no signed byte is below -128)
    a = tm.query_lines(sym, k, canonical, model[0], model[1]).split(b"\n")
    b = tm.query_lines(sym, k, canonical, got[0], got[1]).split(b"\n")
    for i, (x, y) in enumerate(zip(a, b)):
        if x != y:
            return "k-mer %d: model %s, engine %s" % (i, x.decode(), y.decode())
    known = set(tm.as_ints(tm.counts(sym, k, canonical)[0]))
    extra = [x for x in tm.as_ints(got[0]) if x not in known]
    return "the engine holds %d keys that no k-mer of the text has, e.g. %s" % (len(extra), int_to_mer(extra[0], k) if extra else None)


def _check_dump(body, k, canonical, text, min_qual, model, label):
    keys, cnt = model[0], model[1]
    gk, gc = tm.records_to_words(body, k, 8)
    same = len(gk) == len(keys) and np.array_equal(gk, keys) and np.array_equal(gc, cnt)
    assert same, "%s: %d distinct in the dump, model %d; %s" % (label, len(gk), len(keys), _first_diff(text, k, canonical, min_qual, (keys, cnt), (gk, gc)))


def _check(hc, k, canonical, text, min_qual, model, label):
    st = hc.done()
    keys, cnt, n = model
    _check_dump(hc.dump_records(out_counter_len=8), k, canonical, text, min_qual, model, label)
    assert st["kmers"] == n and st["inserted"] == n and st["distinct"] == len(keys), "%s: stats %s, model %d k-mers %d distinct" % (label, st, n, len(keys))


@functools.lru_cache(maxsize=8)
def _model(text, k, canonical, min_qual):
    sym = tm.symbols(text, min_qual)
    return sym, tm.counts(sym, k, canonical)


def _batch(tile, r):
    """j * tile + r: one tile in front of a short last tile, two in front of a long one (room for the read in front)."""
    r = {"16": 16, "96": 96, "256": 256, "tile-16": tile - 16, "tile": tile}[r]
    return (1 if r < tile - 1024 else 2) * tile + r


@functools.lru_cache(maxsize=4)
def _texts(k, tile, r, full):
    batch = _batch(tile, r)
    return batch, qc.cell_texts(batch, tile, k, qc.aimed_cells(k, Q, full))


def _run(hc, text, device, cuda, label):
    if device:
        t = _device(cuda, text)
        hc.add_device_text(t.data_ptr(), len(text))
        del t
    else:
        hc.add_text(text)


# ---- direct insert (MODE 0) at every key width: extract_kernel<KW, SB, 0, 512> and the wide kernel ----------------------
@pytest.mark.parametrize("r", LAST_TILES)
@pytest.mark.parametrize("k", [21, 33, 63, 64, 65, 100, 128])
def test_direct_insert_batch_ends(k, r, cuda):
    from jellyfish_b200 import HashCounter
    canonical = k % 2 == 1
    batch, texts = _texts(k, sc.TILE_512, r, k == 21 or (k == 65 and r in ("96", "256")))    # (the ends and middles elsewhere)
    for j, (text, placed) in enumerate(texts):
        for mq in (Q, 0):
            _, model = _model(text, k, canonical, mq)
            for device in (True, False):
                label = "k=%d batch %d (last tile %d) -Q %r / %s" % (k, batch, qc.last_tile(batch, sc.TILE_512), chr(mq) if mq else None,
                                                                      "one device call" if device else "add_text")
                with HashCounter(1 << 22, 7, k=k, canonical=canonical, no_partition=True, min_qual=mq, max_batch_bytes=batch) as hc:
                    _run(hc, text, device, cuda, label)
                    _check(hc, k, canonical, text, mq, model, label)


# ---- region records (MODE 2): the FAST tail (k = 21, 2^27 slots) and the general form -----------------------------------
def _region(size, k, **kw):
    from jellyfish_b200 import HashCounter
    hc = HashCounter(size, 7, k=k, canonical=True, part_min_mb=1, **kw)
    assert hc.info()["part_regions"] > 0, hc.info()
    return hc


@pytest.mark.parametrize("r", ["96", "256", "tile"])
@pytest.mark.parametrize("k,size", [(21, 1 << 27), (31, 1 << 24), (63, 1 << 24)])
def test_region_records_batch_ends(k, size, r, cuda):
    """Host feeds in batches of the 1024-thread tile geometry (-Q cuts them behind whole records, the default parser at
    the batch length), and device text under the smallest record pool, whose batches are whole tiles."""
    batch, texts = _texts(k, sc.TILE_1024, r, False)
    text, placed = texts[0]
    for mq in (Q, 0):
        _, model = _model(text, k, True, mq)
        label = "region k=%d batch %d -Q %r" % (k, batch, chr(mq) if mq else None)
        with _region(size, k, min_qual=mq, max_batch_bytes=batch) as hc:
            hc.add_text(text)
            _check(hc, k, True, text, mq, model, label + " / add_text")
        with _region(size, k, min_qual=mq, pool_bytes=1) as hc:
            _run(hc, text, True, cuda, label)
            _check(hc, k, True, text, mq, model, label + " / device, smallest record pool")


@pytest.mark.parametrize("k,size", [(21, 1 << 27), (31, 1 << 24)])
def test_region_device_batch_of_512mb(k, size, cuda):
    """Region records take device text in batches of 512 MB, whose last tile is 256 bytes: one cell at byte 512 MB of a
    text of 512 MB + 64 KB.  The filler reads fail the filter, so the model is that of the cell's two reads alone."""
    E = 512 << 20
    c = qc.cell(-30, low=[-5, -17])
    text, body, place = qc.one_cell_text(E, sc.TILE_1024, k, c, E + (64 << 10))
    assert qc.carry_is_rebuilt(place, k, Q, E, sc.TILE_1024)
    _, model = _model(body, k, True, Q)
    t = _device(cuda, text)
    del text
    try:
        with _region(size, k, min_qual=Q) as hc:
            hc.add_device_text(t.data_ptr(), E + (64 << 10))
            _check(hc, k, True, body, Q, model, "region k=%d, one device call over a 512 MB batch end" % k)
    finally:
        del t
        cuda.cuda.empty_cache()


# ---- the neighbours of -Q ---------------------------------------------------------------------------------------------
def test_if_region_prime_unfiltered_update_filtered(cuda):
    """`count --if` in region mode: PRIME reads its text without the filter, UPDATE with it."""
    from jellyfish_b200 import HashCounter
    k = 21
    batch, texts = _texts(k, sc.TILE_1024, "256", False)
    text = texts[0][0]
    prime = tm.counts(tm.symbols(text), k, True)[0]
    _, (uk, uc, _n) = _model(text, k, True, Q)
    cnt = np.zeros(len(prime), np.int64)
    at = {x: i for i, x in enumerate(tm.as_ints(prime))}
    for x, c in zip(tm.as_ints(uk), uc):
        if x in at:
            cnt[at[x]] = c
    assert cnt.sum() and (cnt == 0).any()
    for device in (False, True):
        with _region(1 << 27, k, min_qual=Q, max_batch_bytes=batch) as hc:
            for op in (HashCounter.OP_PRIME, HashCounter.OP_UPDATE):
                hc.set_op(op)
                _run(hc, text, device, cuda, "")
            hc.done()
            _check_dump(hc.dump_records(out_counter_len=8), k, True, text, 0, (prime, cnt), "--if, %s" % ("device" if device else "add_text"))


def test_fasta_fastq_fasta_files(cuda):
    """FASTA, FASTQ, FASTA files in one engine under -Q: every FASTA base passes, no k-mer spans two files."""
    from jellyfish_b200 import HashCounter
    k = 31
    batch, texts = _texts(k, sc.TILE_512, "96", False)
    fq = texts[0][0]
    fa1, _ = sc.dense_text(sc.fasta_events(k, 0), 300000, seed=4)
    fa2, _ = sc.dense_text(sc.fasta_events(k, 0), 200000, seed=5)
    files = [fa1, fq, fa2]
    sym = tm.stream(files, Q)
    model = tm.counts(sym, k, True)
    for device in (True, False):
        with HashCounter(1 << 22, 7, k=k, canonical=True, no_partition=True, min_qual=Q, max_batch_bytes=batch) as hc:
            for f in files:
                _run(hc, f, device, cuda, "")
            _check(hc, k, True, files, Q, model, "FASTA, FASTQ, FASTA / %s" % ("device" if device else "add_text"))


@pytest.mark.parametrize("k", [21, 65])
def test_query_ignores_min_qual(k, cuda):
    """A query reads its text without qualities: query_text on an engine with min_qual gives the unfiltered k-mers, looked
    up in the filtered counts."""
    from jellyfish_b200 import HashCounter
    batch, texts = _texts(k, sc.TILE_512, "256", False)
    text = texts[0][0]
    _, (keys, cnt, _) = _model(text, k, True, Q)
    want = tm.query_lines(tm.symbols(text), k, True, keys, cnt)
    t = _device(cuda, text)
    with HashCounter(1 << 22, 7, k=k, canonical=True, no_partition=True, min_qual=Q, max_batch_bytes=batch) as hc:
        hc.add_device_text(t.data_ptr(), len(text))
        hc.done()
        got = hc.query_text(text)
    if got != want:
        a, b = want.split(b"\n"), got.split(b"\n")
        i = next((i for i, (x, y) in enumerate(zip(a, b)) if x != y), min(len(a), len(b)))
        pytest.fail("query k=%d: %d lines, model %d; first difference at line %d: %r vs model %r" % (
            k, len(b) - 1, len(a) - 1, i, b[i] if i < len(b) else None, a[i] if i < len(a) else None))


def test_region_feed_split_inside_records(cuda):
    """Feed calls cut inside records, next to every cell: the engine carries the open record to the next call."""
    k = 21
    batch, texts = _texts(k, sc.TILE_1024, "256", False)
    text, placed = texts[0]
    _, model = _model(text, k, True, Q)
    cuts = sorted({p["E"] + d for p in placed for d in (-7, 0, 3)} | {p["hs"] + 1 for p in placed} | {p["q2"] + 2 for p in placed})
    cuts = [c for c in cuts if 0 < c < len(text)]
    with _region(1 << 27, k, min_qual=Q, max_batch_bytes=batch) as hc:
        for a, b in zip([0] + cuts, cuts + [len(text)]):
            hc.add_text(text[a:b], begin=a == 0, end=b == len(text))
        _check(hc, k, True, text, Q, model, "region, add_text split at %d cuts inside records" % len(cuts))


def test_record_larger_than_the_batch(cuda):
    """-Q host feeds cut their batches behind whole records: a record longer than the staging batch gives the documented
    error, not a count."""
    from jellyfish_b200 import HashCounter, JellyfishError
    import random
    rng = random.Random(7)
    reads = [qc.record(b"a", sc.bases(100, rng), b"I" * 100), qc.record(b"b", sc.bases(5000, rng), b"I" * 5000),
             qc.record(b"c", sc.bases(100, rng), b"I" * 100)]
    text = b"".join(reads)
    with HashCounter(1 << 16, 7, k=21, canonical=True, no_partition=True, min_qual=Q, max_batch_bytes=4096) as hc:
        with pytest.raises(JellyfishError, match="a record is larger than the staging buffer"):
            hc.add_text(text)
