"""The extraction pipeline's text parsing (K0a nl_scan, K0b tile_state, K1 extract) against the numpy model of the text
contract (tests/text_model.py, itself pinned to the oracle by tests/test_text_model_cpu.py), on the seam corpus
(tests/seam_corpus.py).  The FASTA seam texts put every event at every offset of the chosen range around the window
starts and around the K0a splits, and events in turn at the staging-batch ends; feed-call cuts are taken next to the
placed events.  The dense texts and the FASTQ texts reach the seams at moving, not aimed, offsets.

Every count case checks the exact (key, count) multiset of the dump and the statistics; the forms are one add_device_text
call, add_text through a small staging buffer, add_text split at seam-adjacent cuts, and in region mode the smallest
record pool.  Query cases check `query_text` byte for byte, which pins every k-mer's position.  A failure names the corpus,
the form and the first k-mer (in input order) whose count differs.

K1 instantiations reached (jf_engine.cu run_batch; extract_kernel<KW, SB, MODE, NTH, FAST, NPR>, four-word keys from
jf_wide.cu), as listed by the CUDA profiler for these cases:
  <1, 32|64, 0, 512>, <2, 64|128, 0, 512>, <4, 320, 0, 512>     direct insert, k = 21/31, 33/63/64, 65/128
  <1, 32, 2, 1024, true, 2>                                    region records, FAST tail (k = 21, 2^27 slots)
  <1, 64, 2, 1024, false>, <2, 128, 2, 1024, false>            region records, general form (k = 31, 63)
  <1, 64, 1, 512>, <2, 64, 1, 512>, <4, 320, 1, 512>           route to two shards (k = 21, 33, 65)
  <1, 32, 2, 1024, true, 2> by owner                           record exchange, two shards on one device
  <1, 64, 3, 512>, <2, 64, 3, 512>, <4, 64, 3, 512>            query (k = 21, 33, 65)
The FAST tails with six parity rows (<1, SB, 2, 1024, true, 6>, region records and record exchange) take a table of at
least 2^35 slots of 4 bytes (the parity rows are the position bits above 32: jf_engine.cu table_setup), 128 GB, which
no single device holds; they are not reached here."""
import functools

import numpy as np
import pytest

import seam_corpus as sc
import text_model as tm

pytestmark = pytest.mark.gpu

BATCH = 4 * sc.TILE_512          # staging batch of the host-fed forms: its tile starts are those of the one-call form
BATCH_1024 = 4 * sc.TILE_1024


@pytest.fixture(scope="module")
def cuda(built):
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    torch.cuda.set_device(0)
    return torch


def _device(torch, data):
    t = torch.zeros(len(data) + 16, dtype=torch.uint8, device="cuda")
    if data:
        t[:len(data)] = torch.frombuffer(bytearray(data), dtype=torch.uint8).cuda()
    return t


def _first_diff(sym, k, canonical, model, got):
    """Index (in input order) and line of the first k-mer whose count in `got` differs from the model's."""
    a = tm.query_lines(sym, k, canonical, model[0], model[1]).split(b"\n")
    b = tm.query_lines(sym, k, canonical, got[0], got[1]).split(b"\n")
    for i, (x, y) in enumerate(zip(a, b)):
        if x != y:
            return "k-mer %d: model %s, engine %s" % (i, x.decode(), y.decode())
    return "no k-mer of the text differs (the engine holds keys the text does not)"


def _check_dump(body, k, canonical, sym, model, label):
    keys, cnt, n = model
    gk, gc = tm.records_to_words(body, k, 8)
    same = len(gk) == len(keys) and np.array_equal(gk, keys) and np.array_equal(gc, cnt)
    assert same, "%s: %d distinct in the dump, model %d; %s" % (label, len(gk), len(keys), _first_diff(sym, k, canonical, (keys, cnt), (gk, gc)))


def _check(hc, k, canonical, sym, model, label):
    st = hc.done()
    keys, cnt, n = model
    _check_dump(hc.dump_records(out_counter_len=8), k, canonical, sym, model, label)
    assert st["kmers"] == n and st["inserted"] == n and st["distinct"] == len(keys), "%s: stats %s, model %d k-mers %d distinct" % (label, st, n, len(keys))


@functools.lru_cache(maxsize=6)
def _model(text, k, canonical):
    sym = _symbols(text)
    return sym, tm.counts(sym, k, canonical)


@functools.lru_cache(maxsize=4)
def _symbols(text):
    return tm.symbols(text)


def _feeds(torch, make, text, placed, k, canonical, label, batch, device=True, batched=True, split=True):
    """Count `text` through every feed form with fresh engines from make(**kw)."""
    sym, model = _model(text, k, canonical)
    if device:
        t = _device(torch, text)
        with make() as hc:
            hc.add_device_text(t.data_ptr(), len(text))
            _check(hc, k, canonical, sym, model, "%s / one device call" % label)
        del t
    if batched:
        with make(max_batch_bytes=batch) as hc:
            hc.add_text(text)
            _check(hc, k, canonical, sym, model, "%s / add_text in %d-byte batches" % (label, sc.batch_len(batch)))
    if split:
        cuts = sc.split_points(text, [p + d for i, (p, _) in enumerate(placed[:400]) for d in ((i % 5) - 2, k - 1 + i % 3)])
        with make(max_batch_bytes=batch) as hc:
            for a, b in zip([0] + cuts, cuts + [len(text)]):
                hc.add_text(text[a:b], begin=a == 0, end=b == len(text))
            _check(hc, k, canonical, sym, model, "%s / add_text split at %d cuts" % (label, len(cuts)))


def _offsets(k):
    """Every offset in [-(k+2), k+2] for k = 21; for the other k the ends and the middle of that range."""
    if k == 21:
        return None
    return sorted(set(list(range(-(k + 2), -(k - 3))) + list(range(-3, 4)) + list(range(k - 3, k + 3))))


@functools.lru_cache(maxsize=None)
def _seam_texts(k, tile, batch):
    # (the '\r' run as long as a batch has its own test below)
    return sc.seam_texts(k, tile, sc.fasta_events(k, 0), batch=batch, offs=_offsets(k))


# ---- direct insert (MODE 0) at every key width: extract_kernel<KW, SB, 0, 512> and the wide kernel ----------------------
@pytest.mark.parametrize("k", [21, 31, 33, 63, 64, 65, 128])
def test_direct_insert_seams(k, cuda):
    from jellyfish_b200 import HashCounter
    canonical = k % 2 == 1
    for j, (text, placed) in enumerate(_seam_texts(k, sc.TILE_512, BATCH)):
        def make(**kw):
            return HashCounter(1 << 22, 7, k=k, canonical=canonical, no_partition=True, **kw)
        _feeds(cuda, make, text, placed, k, canonical, "seams k=%d text %d (%s .. %s)" % (k, j, placed[0][1], placed[-1][1]), BATCH,
               batched=j < (2 if k == 21 else 1), split=j == 0)


@pytest.mark.parametrize("k", [21, 65])
def test_direct_insert_dense(k, cuda):
    from jellyfish_b200 import HashCounter
    text, placed = sc.dense_text(sc.fasta_events(k, 0), 3 << 20)
    _feeds(cuda, lambda **kw: HashCounter(1 << 22, 7, k=k, canonical=True, no_partition=True, **kw), text, placed, k, True,
           "dense k=%d" % k, 65536 + 13)            # (a batch of 65552 bytes: the engine rounds up to 16)


# ---- region records (MODE 2): the FAST tail with two parity rows (k21 bench geometry) and the general form --------------
@pytest.mark.parametrize("k,size", [(21, 1 << 27), (31, 1 << 24), (63, 1 << 24)])
def test_region_records_seams(k, size, cuda):
    from jellyfish_b200 import HashCounter

    def make(**kw):
        hc = HashCounter(size, 7, k=k, canonical=True, part_min_mb=1, **kw)
        assert hc.info()["part_regions"] > 0, hc.info()
        return hc
    for j, (text, placed) in enumerate(_seam_texts(k, sc.TILE_1024, BATCH_1024)[:2 if k == 21 else 1]):
        label = "region k=%d text %d" % (k, j)
        _feeds(cuda, make, text, placed, k, True, label, BATCH_1024, split=j == 0 and k == 21)
        if j == 0:
            sym, model = _model(text, k, True)
            t = _device(cuda, text)
            with make(pool_bytes=1) as hc:                   # the host cuts the text to what an empty arena takes
                hc.add_device_text(t.data_ptr(), len(text))
                _check(hc, k, True, sym, model, "%s / smallest record pool" % label)


# ---- route (MODE 1): keys bucketed by owning shard, inserted by two shard engines on one device ------------------------
@pytest.mark.parametrize("k", [21, 33, 65])
def test_route_two_shards_seams(k, cuda):
    """Every k-mer lands in the bucket of its owner: the buckets inserted into the owners' engines must dump, together,
    the model's counts."""
    torch = cuda
    from jellyfish_b200 import HashCounter
    world = 2
    text, placed = _seam_texts(k, sc.TILE_512, BATCH)[0]
    sym, model = _model(text, k, True)
    t = _device(torch, text)
    cap = len(text)                                          # one k-mer per byte at most
    for batch in (0, BATCH):
        label = "route k=%d batch %d" % (k, sc.batch_len(batch))
        shards = [HashCounter(1 << 22, 7, k=k, canonical=True, shard_index=r, n_shards=world, allow_regrow=False, no_partition=True,
                              max_batch_bytes=batch) for r in range(world)]
        try:
            kw = shards[0].key_words
            send = torch.zeros((world, cap * kw), dtype=torch.int64, device="cuda")
            counts = torch.zeros(world, dtype=torch.int64, device="cuda")
            shards[0].extract_route(t.data_ptr(), len(text), send.data_ptr(), cap, counts.data_ptr())
            torch.cuda.synchronize()
            c = counts.tolist()
            assert sum(c) == model[2], "%s: %d keys routed, model %d k-mers" % (label, sum(c), model[2])
            body = b""
            for d in range(world):
                if c[d]:
                    shards[d].insert_keys(send[d].data_ptr(), c[d])
                shards[d].done()
                body += shards[d].dump_records(out_counter_len=8)
            _check_dump(body, k, True, sym, model, label)
        finally:
            for hc in shards:
                hc.close()


# ---- record exchange (MODE 2 by owner): jfgpu_shard_* with two shards on one device -----------------------------------
def test_record_exchange_seams(cuda):
    """K1 files region records of the global table by owning shard; the chunks are copied into the owners' receive pools
    the way the all-to-all would, re-filed and drained; the shards' dumps together must be the model's counts.  The text
    goes through in device calls cut next to seams (16-byte aligned, never inside a '\r' run)."""
    torch = cuda
    from jellyfish_b200 import HashCounter
    from jellyfish_b200.distributed import CHUNK
    k, world, size = 21, 2, 1 << 27
    text, placed = _seam_texts(k, sc.TILE_1024, BATCH_1024)[0]
    sym, model = _model(text, k, True)
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    arena = 2 * n_sm * max(1, 1024 // world) + 64
    torch.cuda.empty_cache()
    shards, bufs = [], []
    try:
        for r in range(world):
            hc = HashCounter(size, 7, k=k, canonical=True, shard_index=r, n_shards=world, allow_regrow=False, part_min_mb=1,
                             pool_bytes=2 << 30, max_batch_bytes=1 << 20)
            shards.append(hc)
            send = torch.empty(2 * world * arena * CHUNK, dtype=torch.uint8, device="cuda")
            send_dir = torch.empty(2 * world * arena * 8, dtype=torch.uint8, device="cuda")
            recv = torch.empty(world * arena * CHUNK, dtype=torch.uint8, device="cuda")
            recv_dir = torch.empty(world * arena * 8, dtype=torch.uint8, device="cuda")
            assert hc.shard_setup(send.data_ptr(), send_dir.data_ptr(), arena, recv.data_ptr(), recv_dir.data_ptr(), arena)
            bufs.append((send, send_dir, recv, recv_dir))
        buf = _device(torch, text)
        cuts = []
        for p, _ in placed[::3]:                             # device calls cut next to the placed events
            c = (p + 7) & ~15
            while 0 < c < len(text) and text[c - 1] == 13:
                c -= 16
            if 0 < c < len(text) and (not cuts or c > cuts[-1]):
                cuts.append(c)
        bounds = list(zip([0] + cuts, cuts + [len(text)]))
        for i, (a, b) in enumerate(bounds):
            bank = i & 1
            shards[0].shard_extract(buf.data_ptr() + a, b - a, bank, begin=a == 0, end=b == len(text))
            counts = shards[0].shard_pack(bank)
            assert max(counts) <= arena
            send, send_dir = bufs[0][0], bufs[0][1]
            for d in range(world):
                c = counts[d]
                recv, recv_dir = bufs[d][2], bufs[d][3]
                a0 = (bank * world + d) * arena
                recv[:c * CHUNK] = send[a0 * CHUNK:(a0 + c) * CHUNK]
                recv_dir[:c * 8] = send_dir[a0 * 8:(a0 + c) * 8]
                torch.cuda.synchronize()
                got = [0] * world
                got[0] = c
                shards[d].shard_unpack(got)
                torch.cuda.synchronize()
        body = b""
        n_ins = 0
        for hc in shards:
            n_ins += hc.done()["inserted"]
            body += hc.dump_records(out_counter_len=8)
        assert n_ins == model[2], "record exchange: %d inserted, model %d k-mers (%d device calls)" % (n_ins, model[2], len(bounds))
        _check_dump(body, k, True, sym, model, "record exchange, %d device calls" % len(bounds))
    finally:
        for hc in shards:
            hc.close()
        torch.cuda.empty_cache()


# ---- query (MODE 3): byte for byte, every position --------------------------------------------------------------------
@pytest.mark.parametrize("k", [21, 33, 65])
def test_query_seams_byte_for_byte(k, cuda):
    from jellyfish_b200 import HashCounter
    text, placed = _seam_texts(k, sc.TILE_512, BATCH)[0]
    sym, (keys, cnt, _) = _model(text, k, True)
    want = tm.query_lines(sym, k, True, keys, cnt)
    t = _device(cuda, text)
    for batch in (0, BATCH):
        with HashCounter(1 << 22, 7, k=k, canonical=True, no_partition=True, max_batch_bytes=batch) as hc:
            hc.add_device_text(t.data_ptr(), len(text))
            hc.done()
            got = hc.query_text(text)
        if got != want:
            a, b = want.split(b"\n"), got.split(b"\n")
            i = next((i for i, (x, y) in enumerate(zip(a, b)) if x != y), min(len(a), len(b)))
            pytest.fail("query k=%d batch %d: %d lines, model %d; first difference at line %d: %r vs model %r" % (
                k, batch, len(b) - 1, len(a) - 1, i, b[i] if i < len(b) else None, a[i] if i < len(a) else None))


# ---- the '\r' run that fills a staging batch ---------------------------------------------------------------------------
@pytest.mark.parametrize("after", [b"ACGTTGCA", b"\nACGTTGCA", b"\r\nACG", b""])
def test_cr_run_filling_a_batch(after, cuda):
    """A run of '\\r' as long as the staging batch, or one byte then such a run, must give what one call gives: reset the
    window when a base follows it, be dropped when a line end follows it."""
    from jellyfish_b200 import HashCounter
    import random
    k, batch = 11, 4096
    for lead in (b"", b"T"):
        # the first batch is one sequence line that ends in a base: the run is in the middle of a line
        text = b">x\n" + sc.bases(batch - 3, random.Random(1)) + lead + b"\r" * batch + after + b"GATTACAGATTACA\n"
        sym = tm.symbols(text)
        model = tm.counts(sym, k, False)
        with HashCounter(1 << 16, 7, k=k, max_batch_bytes=batch) as hc:
            hc.add_text(text)
            _check(hc, k, False, sym, model, "cr run of %d after %r before %r" % (batch, lead, after))
        keys, cnt, _ = model
        with HashCounter(1 << 16, 7, k=k, max_batch_bytes=batch) as hc:
            hc.add_text(text)
            hc.done()
            assert hc.query_text(text) == tm.query_lines(sym, k, False, keys, cnt)


def test_calls_split_inside_dos_line_ends(cuda):
    """Feed calls that end between a line's '\\r' run and its '\\n': the end of a call is a line end, so the lines still
    join (a base after the run would reset the window; a call never ends on a run that a base follows)."""
    import random
    from jellyfish_b200 import HashCounter
    k = 31
    rng = random.Random(3)
    text = b">x\r\n" + b"".join(sc.bases(rng.randrange(1, 90), rng) + b"\r" * rng.choice((1, 1, 2, 300)) + b"\n" for _ in range(3000))
    runs = [i for i in range(1, len(text)) if text[i] == 10 and text[i - 1] == 13]
    cuts = sc.split_points(text, [r - d for r in runs[::7] for d in (0, 1)])
    assert any(text[c - 1] == 13 for c in cuts)
    sym = tm.symbols(text)
    model = tm.counts(sym, k, True)
    for batch in (0, 4096):
        with HashCounter(1 << 20, 7, k=k, canonical=True, no_partition=True, max_batch_bytes=batch) as hc:
            for a, b in zip([0] + cuts, cuts + [len(text)]):
                hc.add_text(text[a:b], begin=a == 0, end=b == len(text))
            _check(hc, k, True, sym, model, "DOS line ends split between '\\r' and '\\n' (batch %d)" % batch)


# ---- FASTQ and -Q ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("k,eol", [(31, b"\n"), (31, b"\r\n"), (65, b"\r\n")])
def test_fastq(k, eol, cuda):
    from jellyfish_b200 import HashCounter
    text = sc.fastq_text(3 << 20, k, seed=k, eol=eol, long_every=97)
    placed = [(p, "record") for p in range(0, len(text), 7919)]
    _feeds(cuda, lambda **kw: HashCounter(1 << 22, 7, k=k, canonical=True, no_partition=True, **kw), text, placed, k, True,
           "fastq k=%d eol=%r" % (k, eol), BATCH)


@pytest.mark.parametrize("form", ["fastq", "fastq_dos", "fasta"])
def test_min_quality(form, cuda):
    from jellyfish_b200 import HashCounter
    k, q = 21, ord("5")
    if form == "fasta":
        text, _ = sc.dense_text(sc.fasta_events(k, 0), 1 << 20)
    else:
        text = sc.fastq_text(2 << 20, k, seed=9, eol=b"\r\n" if form == "fastq_dos" else b"\n", low=b"!#4\x80\xf0", long_every=0)
    sym = tm.symbols(text, q)
    model = tm.counts(sym, k, True)
    t = _device(cuda, text)
    with HashCounter(1 << 22, 7, k=k, canonical=True, no_partition=True, min_qual=q) as hc:
        hc.add_device_text(t.data_ptr(), len(text))
        _check(hc, k, True, sym, model, "-Q %s / one device call" % form)
    with HashCounter(1 << 22, 7, k=k, canonical=True, no_partition=True, min_qual=q, max_batch_bytes=BATCH) as hc:
        for a in range(0, len(text), 300007):                # feed calls cut anywhere: the engine keeps the open record
            hc.add_text(text[a:a + 300007], begin=a == 0, end=a + 300007 >= len(text))
        _check(hc, k, True, sym, model, "-Q %s / add_text split" % form)


# ---- file ends at a seam -----------------------------------------------------------------------------------------------
def test_file_ends_at_seams(cuda):
    from jellyfish_b200 import HashCounter
    k = 31
    text, placed = sc.dense_text(sc.fasta_events(k, 0), 200000)
    ends = [s + d for s, _ in sc.seams(sc.TILE_512, len(text))[:6] for d in (-k - 1, -1, 0, 1, k)]
    files = [text[:e] for e in ends if 0 < e < len(text)] + [b"", b">only a header", b">h\nACGT\r\r\r"]
    sym = tm.stream(files)
    model = tm.counts(sym, k, True)
    with HashCounter(1 << 22, 7, k=k, canonical=True, no_partition=True) as hc:
        for f in files:
            t = _device(cuda, f)
            hc.add_device_text(t.data_ptr(), len(f))
        _check(hc, k, True, sym, model, "file ends / device")
    with HashCounter(1 << 22, 7, k=k, canonical=True, no_partition=True, max_batch_bytes=BATCH) as hc:
        for f in files:
            hc.add_text(f)
        _check(hc, k, True, sym, model, "file ends / add_text")
