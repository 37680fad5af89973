"""A cleared table is zero in meaning only until its first drain, which writes every window of the table without reading it
(jf_engine.cu table_zero / table_materialize, jf_window.cuh WinDev::lazy_win).  These tests leave stale counts in the slots, clear,
and hold what the engine reports afterwards to the C restatement's database for the same input.

The table: k=17, 2^23 slots of 32 bits, 256 regions of 2^15 slots (two windows each), 4-byte records, i.e. the window form
of K2 under part_min_mb=1.  With 1 MB batches a group of the drain holds about three regions, so a drain has dozens of
groups."""
import os

import numpy as np
import pytest

import jfutil

pytestmark = pytest.mark.gpu

K, SIZE, SIZE_ARG = 17, 8_000_000, "8M"
WIN_SLOTS = 1 << 14


@pytest.fixture(scope="module")
def lazy_inputs(built, workdir):
    """name -> (fasta path, oracle header, oracle body).  A fills the table to 0.86, B to 0.36, C holds 8 k-mers (most
    regions and a whole group of them receive nothing), G has more distinct k-mers than the table has slots, S is 30 Mbp of
    a period-3 repeat between two random megabases."""
    import gen
    out = {}
    seqs = {"A": gen._seq(7_200_000, 501), "B": gen._seq(3_000_000, 503), "C": gen._seq(24, 504), "G": gen._seq(9_500_000, 502),
            "S": gen._seq(1_000_000, 505) + b"ACG" * 10_000_000 + gen._seq(1_000_000, 506)}
    for name, seq in seqs.items():
        fa = os.path.join(workdir, "lazy_%s.fa" % name)
        with open(fa, "wb") as f:
            f.write(gen.fasta(seq))
        db = os.path.join(workdir, "lazy_%s.jf" % name)
        jfutil.run([jfutil.ORACLE_C, "count", "-m", str(K), "-s", SIZE_ARG, "-C", "-o", db, fa])
        h, b = jfutil.split_db(db)
        out[name] = (fa, h, b)
    return out


def _counter(**kw):
    from jellyfish_b200 import HashCounter
    hc = HashCounter(SIZE, 7, k=K, canonical=True, part_min_mb=1, pool_bytes=1 << 30, max_batch_bytes=1 << 20, **kw)
    info = hc.info()
    assert info["lsize"] == 23 and info["slot_bits"] == 32 and info["part_regions"] == 256 and info["part_rec_bytes"] == 4
    return hc


def _count_and_check(hc, inp):
    fa, h, b = inp
    hc.add_files([fa])
    st = hc.done()
    assert st["kmers"] == st["inserted"]
    assert hc.dump_records() == b
    hdr = hc.header()
    assert {x: hdr[x] for x in jfutil.SEMANTIC_KEYS} == jfutil.semantic(h)
    return st


def _empty(hc, probe_keys):
    assert hc.get_many(probe_keys) == [0] * len(probe_keys)
    assert hc.histogram(16) == [0] * 16
    assert hc.dump_records() == b""
    st = hc.done()
    assert st["inserted"] == st["distinct"] == 0


def _positions(header, key):
    """Original positions of the keys (RectangularBinaryMatrix::times, as jfutil.hash_pos), vectorised."""
    m = header["matrix1"]
    assert not m["identity"]
    pos = np.zeros(len(key), np.uint64)
    for i in range(m["c"]):
        pos ^= ((key >> np.uint64(i)) & np.uint64(1)) * np.uint64(m["columns"][m["c"] - 1 - i])
    return pos & np.uint64(header["size"] - 1)


def _keys(header, body):
    kb = (header["key_len"] + 7) // 8
    a = np.frombuffer(body, np.uint8).reshape(-1, kb + header["counter_len"])
    key = np.zeros(len(a), np.uint64)
    for j in range(kb):
        key |= a[:, j].astype(np.uint64) << np.uint64(8 * j)
    return key


def test_reuse_after_clear(lazy_inputs):
    """Count A, clear, count B: nothing of A may survive.  Then B once more after a clear."""
    with _counter() as hc:
        _count_and_check(hc, lazy_inputs["A"])
        hc.clear()
        st1 = _count_and_check(hc, lazy_inputs["B"])
        hc.clear()
        st2 = _count_and_check(hc, lazy_inputs["B"])
        assert (st1["kmers"], st1["distinct"]) == (st2["kmers"], st2["distinct"])


def test_nothing_fed_after_clear_and_on_a_fresh_counter(lazy_inputs):
    """clear() then nothing: lookup, histogram, dump and done see an empty table (no drain ever wrote it).  The same on a
    counter just created, whose memory is what the previous counter left."""
    fa, h, b = lazy_inputs["A"]
    probe = [int(x) for x in _keys(h, b)[:: 100_000]]
    with _counter() as hc:
        _count_and_check(hc, lazy_inputs["A"])
        hc.clear()
        _empty(hc, probe)
    with _counter() as hc:
        _empty(hc, probe)
        _count_and_check(hc, lazy_inputs["B"])


def test_sparse_input_after_clear(lazy_inputs):
    """8 k-mers after a full table: nearly every region, and all 64 regions of one group of the drain, get no record (the
    group is zeroed without any window kernel)."""
    fa, h, b = lazy_inputs["C"]
    regions = set((_positions(h, _keys(h, b)) >> np.uint64(15)).tolist())
    assert len(regions) <= 8 and any(all(r not in regions for r in range(g, g + 64)) for g in range(0, 256, 64))
    with _counter() as hc:
        _count_and_check(hc, lazy_inputs["A"])
        hc.clear()
        st = _count_and_check(hc, lazy_inputs["C"])
        assert st["distinct"] == len(b) // 9


def test_deferred_records_across_group_boundaries(lazy_inputs):
    """0.86 load: keys whose probes leave their window in shared memory go to the global path.  For many windows that end a
    region, and so possibly a group, more distinct keys hash into their last s slots than those s slots hold, so some
    key of them must leave the window into the next one, which a write-only drain writes without reading."""
    fa, h, b = lazy_inputs["A"]
    with _counter() as hc:
        _count_and_check(hc, lazy_inputs["A"])
        hdr = hc.header()
        pos = _positions(hdr, _keys(h, b))
        assert np.all(np.diff(pos.astype(np.int64)) >= 0)           # the host hash is the one the dump is ordered by
        win, local = (pos >> np.uint64(14)).astype(np.int64), (pos & np.uint64(WIN_SLOTS - 1)).astype(np.int64)
        n_win = hdr["size"] // WIN_SLOTS
        forced = np.zeros(n_win, bool)
        for s in range(1, 64):
            forced |= np.bincount(win[local >= WIN_SLOTS - s], minlength=n_win) > s
        assert forced[1::2].sum() >= 64                            # (two windows per region)
        hc.clear()
        _count_and_check(hc, lazy_inputs["A"])


def test_regrow_in_the_middle_of_a_write_only_drain(lazy_inputs):
    """More distinct k-mers than slots: the table doubles while the first drain after a clear is under way; header (size,
    matrix) and body as the restatement's."""
    with _counter() as hc:
        _count_and_check(hc, lazy_inputs["A"])
        hc.clear()
        st = _count_and_check(hc, lazy_inputs["G"])
        assert st["regrows"] >= 1 and hc.info()["lsize"] == 24


def test_full_spill_list_before_the_first_drain(lazy_inputs):
    """30 Mbp of a period-3 repeat: its k-mers fall into at most three regions, so a pass of K1 (4096 k-mers per CTA) can put at
    most 3 x 128 of them into region rings and chunks and spills the rest -- about 27 M k-mers, beyond the 16 M of the
    spill list, all before the first drain.  K1 inserts the overflow into the table itself, which is not in memory yet:
    the windows those insertions reach are zeroed first, and the drain keeps them.  On a fresh counter and after a clear
    (stale counts in the slots)."""
    with _counter() as hc:
        _count_and_check(hc, lazy_inputs["S"])
        hc.clear()
        _count_and_check(hc, lazy_inputs["S"])
