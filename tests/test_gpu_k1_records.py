"""K1's region records at the k21 geometry of the bench, counted exactly against the sort-based model (tests/kmer_model.py).

k=21 into 2^27 slots of 32 bits under part_min_mb=1: 1024 regions of 2^17 slots and 4-byte records, so K1 takes its FAST
tail -- records staged in one shared-memory ring per region, a ring pass after every 8 k-mers per thread, chunks taken from
the CTA's arena through a cursor kept in shared memory for the launch.  Every case compares the statistics, the count
histogram and the counts of the sampled input k-mers and of random keys with the model's.

  one launch     200 Mbp from device memory in one K1 launch: every CTA closes and opens about 750 chunks
  many launches  the same text from host memory in 8 MB batches: dozens of launches share each arena between two
                 drains, each one starting from the cursor the one before left
  small pool     the smallest record pool (two chunks per region and CTA): the host cuts the text so that one launch fits an
                 empty arena and drains before nearly every launch, which resets the cursors
  skewed         short tandem repeats and a poly-A run: rings overflow within a pass, into the spill list and the direct
                 insertion behind it"""
import ctypes as C

import numpy as np
import pytest

import kmer_model as km

pytestmark = pytest.mark.gpu

K, SIZE = 21, 1 << 27
N_SAMPLE, N_RANDOM = 65536, 20000


def _text(dev, parts):
    """A one-record FASTA text (70-column lines) of the concatenated ACGT parts, as a uint8 tensor on `dev`."""
    import torch
    seq = np.concatenate(parts)
    body = np.full(len(seq) + (len(seq) + 69) // 70, ord("\n"), np.uint8)
    idx = np.arange(len(seq))
    body[idx + idx // 70] = seq
    raw = np.concatenate([np.frombuffer(b">k1\n", np.uint8), body, np.full(16, 0, np.uint8)])
    t = torch.from_numpy(raw).to(dev)
    return t, len(raw) - 16, len(seq)


def _random(n, seed):
    return np.frombuffer(b"ACGT", np.uint8)[np.random.default_rng(seed).integers(0, 4, n)]


def _repeat(unit_len, total, seed):
    u = _random(unit_len, seed)
    return np.tile(u, total // unit_len + 1)[:total]


def _queries(text, n_text, n_bases, dev):
    import torch
    starts = np.random.default_rng(7).integers(0, n_bases - K + 1, size=N_SAMPLE, dtype=np.int64)
    base = torch.from_numpy(starts[:, None] + np.arange(K, dtype=np.int64)[None, :]).to(dev)
    sampled = km.mers_words(text[4 + base + base // 70], K)        # base i sits at byte 4 + i + i // 70
    return torch.cat([sampled, km.random_words(N_RANDOM, K, 99, dev)])


def _counter(**kw):
    from jellyfish_b200 import HashCounter
    hc = HashCounter(SIZE, 7, k=K, canonical=True, part_min_mb=1, **kw)
    info = hc.info()
    assert (info["lsize"], info["slot_bits"], info["part_regions"], info["part_rec_bytes"]) == (27, 32, 1024, 4), info
    return hc


def _check(hc, st, model, queries):
    assert st["kmers"] == model.n_kmers and st["inserted"] == st["kmers"], st
    assert st["distinct"] == model.distinct(), (st["distinct"], model.distinct())
    assert hc.histogram(km.N_BINS) == model.histogram()
    words = np.ascontiguousarray(queries.cpu().numpy()).view(np.uint64).reshape(-1)
    got = np.zeros(queries.shape[0], np.uint64)
    hc._check(hc._lib.jfgpu_lookup(hc._h, C.c_void_p(words.ctypes.data), queries.shape[0], C.c_void_p(got.ctypes.data)))
    want = model.query_counts.numpy()
    bad = np.nonzero(got.astype(np.int64) != want)[0]
    assert not len(bad), "%d of %d lookups differ, first at %d (engine %d, model %d)" % (len(bad), len(want), bad[0], got[bad[0]], want[bad[0]])


@pytest.fixture(scope="module")
def uniform(built):
    """200 Mbp: a random 12 Mbp unit repeated (12 M distinct k-mers, about 0.09 of the table), then 8 Mbp of its own."""
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    torch.cuda.set_device(0)
    text, n_text, n_bases = _text("cuda", [_repeat(12_000_000, 192_000_000, 11), _random(8_000_000, 12)])
    q = _queries(text, n_text, n_bases, "cuda")
    model = km.count(text[:n_text], K, queries=q)
    yield text, n_text, model, q
    del text
    torch.cuda.empty_cache()


def test_one_launch_closes_chunks_many_times(uniform):
    text, n_text, model, q = uniform
    with _counter() as hc:
        hc.add_device_text(text.data_ptr(), n_text)
        _check(hc, hc.done(), model, q)
        hc.clear()                                          # and again into the cleared table: the arenas start over
        hc.add_device_text(text.data_ptr(), n_text)
        _check(hc, hc.done(), model, q)


def test_many_launches_between_two_drains(uniform):
    text, n_text, model, q = uniform
    host = text[:n_text].cpu().numpy().tobytes()
    with _counter(pool_bytes=4 << 30, max_batch_bytes=8 << 20) as hc:
        hc.add_text(host)
        _check(hc, hc.done(), model, q)


def test_smallest_record_pool(uniform):
    text, n_text, model, q = uniform
    with _counter(pool_bytes=1) as hc:
        hc.add_device_text(text.data_ptr(), n_text)
        _check(hc, hc.done(), model, q)


def test_skewed_input_overflows_rings(built):
    """Tandem repeats of 40 to 3000 bases put a few regions under a load that overflows their rings within one pass; a
    2 Mbp poly-A run sends one k-mer to one region at every position."""
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    torch.cuda.set_device(0)
    parts = [_random(4_000_000, 21)]
    for i, unit in enumerate((40, 150, 600, 3000)):
        parts += [_repeat(unit, 6_000_000, 30 + i), _random(1_000_000, 40 + i)]
    parts += [np.full(2_000_000, ord("A"), np.uint8), _random(4_000_000, 22)]
    text, n_text, n_bases = _text("cuda", parts)
    q = _queries(text, n_text, n_bases, "cuda")
    model = km.count(text[:n_text], K, queries=q)
    with _counter() as hc:
        hc.add_device_text(text.data_ptr(), n_text)
        _check(hc, hc.done(), model, q)
    with _counter(max_batch_bytes=4 << 20) as hc:
        hc.add_text(text[:n_text].cpu().numpy().tobytes())
        _check(hc, hc.done(), model, q)
