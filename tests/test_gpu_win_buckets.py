"""The window form of K2 places each window's records into a bucket of fixed capacity (jf_window.cuh, win_scatter_kernel<true>)
and falls back to the exact two-pass placement for a group in which some window overflows its bucket.  These tests hold
the database of every path to the C restatement's for the same input:

* k2_mode 0: buckets, fallback only on overflow; 3: every group takes the exact placement; 4: buckets of no slack, so
  nearly every group overflows one and falls back after the bucket pass;
* seconds_win_hist is the time of the exact placement of overflowed groups: 0 for iid input under mode 0, > 0 when a
  fallback ran;
* two geometries at k=17, both in 256 regions: 2^23 slots (two windows per region) and 2^28 slots (64 windows per region)."""
import os

import numpy as np
import pytest

import jfutil

pytestmark = pytest.mark.gpu

K = 17
GEOMETRIES = {"2wpr": dict(size=8_000_000, size_arg="8M", lsize=23), "64wpr": dict(size=1 << 28, size_arg="256M", lsize=28)}


@pytest.fixture(scope="module")
def bucket_inputs(built, workdir):
    """(geometry, name) -> (fasta paths, oracle header, oracle body).  A fills the small table to 0.86; B and D are 3 Mbp
    each and are counted together (BD); R is 30 Mbp of a period-3 repeat between two random megabases."""
    import gen
    seqs = {"A": gen._seq(7_200_000, 601), "B": gen._seq(3_000_000, 603), "D": gen._seq(3_000_000, 607),
            "R": gen._seq(1_000_000, 605) + b"ACG" * 10_000_000 + gen._seq(1_000_000, 606)}
    paths = {}
    for name, seq in seqs.items():
        paths[name] = os.path.join(workdir, "bucket_%s.fa" % name)
        with open(paths[name], "wb") as f:
            f.write(gen.fasta(seq))
    out = {}
    for geometry, g in GEOMETRIES.items():
        for name, files in {"A": ["A"], "BD": ["B", "D"], "R": ["R"]}.items():
            db = os.path.join(workdir, "bucket_%s_%s.jf" % (geometry, name))
            fas = [paths[x] for x in files]
            jfutil.run([jfutil.ORACLE_C, "count", "-m", str(K), "-s", g["size_arg"], "-C", "-o", db] + fas)
            h, b = jfutil.split_db(db)
            out[geometry, name] = (fas, h, b)
    return out


def _counter(geometry, k2_mode):
    from jellyfish_b200 import HashCounter
    g = GEOMETRIES[geometry]
    hc = HashCounter(g["size"], 7, k=K, canonical=True, part_min_mb=1, pool_bytes=1 << 30, max_batch_bytes=1 << 20, k2_mode=k2_mode)
    info = hc.info()
    assert info["lsize"] == g["lsize"] and info["slot_bits"] == 32 and info["part_regions"] == 256 and info["part_rec_bytes"] == 4
    return hc


def _check(hc, inp, feeds=None):
    """Count the files of `inp` (in `feeds` calls of add_files + done), compare with the restatement, return the stats."""
    fas, h, b = inp
    for group in feeds or [fas]:
        hc.add_files(group)
        st = hc.done()
    assert st["kmers"] == st["inserted"]
    assert hc.dump_records() == b
    hdr = hc.header()
    assert {x: hdr[x] for x in jfutil.SEMANTIC_KEYS} == jfutil.semantic(h)
    return st


@pytest.mark.parametrize("geometry", sorted(GEOMETRIES))
def test_bucket_and_exact_placement_agree(bucket_inputs, geometry):
    """Modes 0, 3 and 4 give the restatement's database and the same statistics; only the overflowed groups (none for iid
    input under mode 0, all under 3, nearly all under 4) take the exact placement."""
    seen = {}
    for mode in (0, 3, 4):
        with _counter(geometry, mode) as hc:
            st = _check(hc, bucket_inputs[geometry, "A"])
        seen[mode] = (st["kmers"], st["inserted"], st["distinct"])
        assert st["seconds_win_scatter"] > 0 and st["seconds_win_insert"] > 0
        if mode == 0:
            assert st["seconds_win_hist"] == 0.0
        else:
            assert st["seconds_win_hist"] > 0
    assert seen[0] == seen[3] == seen[4]


def test_hot_window_falls_back_to_the_exact_placement(bucket_inputs):
    """A period-3 repeat puts a large share of its 30 M k-mers into the record pool, all in the windows of its three k-mers.
    In the small table they hash into three different regions (of two windows), so in each of those regions one window
    holds nearly all records and its bucket (about half of them plus the slack) overflows; in the large table a region
    has 64 windows and the bucket about 1/64 of the region's records.  The group overflows under mode 0 too, and the exact
    placement still gives the restatement's database."""
    fas, h, b = bucket_inputs["2wpr", "R"]
    kb = (h["key_len"] + 7) // 8
    a = np.frombuffer(b, np.uint8).reshape(-1, kb + h["counter_len"])
    key, counts = np.zeros(len(a), np.uint64), np.zeros(len(a), np.uint64)
    for j in range(kb):
        key |= a[:, j].astype(np.uint64) << np.uint64(8 * j)
    for j in range(h["counter_len"]):
        counts |= a[:, kb + j].astype(np.uint64) << np.uint64(8 * j)
    hot = np.argsort(counts)[-3:]
    assert int(counts[hot].min()) > 9_000_000                     # the three k-mers of the repeat
    m = h["matrix1"]
    pos = np.zeros(3, np.uint64)
    for i in range(m["c"]):
        pos ^= ((key[hot] >> np.uint64(i)) & np.uint64(1)) * np.uint64(m["columns"][m["c"] - 1 - i])
    pos &= np.uint64(h["size"] - 1)
    assert len(set((pos >> np.uint64(15)).tolist())) == 3
    for geometry in sorted(GEOMETRIES):
        with _counter(geometry, 0) as hc:
            st = _check(hc, bucket_inputs[geometry, "R"])
        assert st["seconds_win_hist"] > 0


@pytest.mark.parametrize("mode", [0, 4])
def test_second_drain_into_a_table_in_memory(bucket_inputs, mode):
    """Feed B, finish, feed D, finish: the second drain loads every window it inserts into (the table is in memory after the
    first), through buckets (mode 0) or through buckets and the fallback (mode 4)."""
    for geometry in sorted(GEOMETRIES):
        fas = bucket_inputs[geometry, "BD"][0]
        with _counter(geometry, mode) as hc:
            st = _check(hc, bucket_inputs[geometry, "BD"], feeds=[[fas[0]], [fas[1]]])
        assert (st["seconds_win_hist"] == 0.0) if mode == 0 else (st["seconds_win_hist"] > 0)


@pytest.mark.parametrize("mode", [0, 4])
def test_2048_windows_per_region(built, mode):
    """2^33 slots at k=17 in 128 MB regions: 256 regions of 2^25 slots, 2048 windows each, the widest geometry
    window_enabled takes (every thread of the bucket pass's scan owns two windows; win_scan sees 131 072 windows in a
    group of 64 regions).  About 200 Mbp of synthetic text, counted after a clear() (a write-only drain), through buckets
    (mode 0) and through buckets without slack and the exact placement (mode 4), against the sort-based model: statistics,
    histogram, sampled lookups and the digest of the whole dump.  (The C restatement cannot hold 2^33 slots.)"""
    import torch
    import kmer_model as km
    from jellyfish_b200 import HashCounter, _lib
    from test_gpu_bench_exact import _check_dump, _check_step, _queries, _synth
    need = 40e9
    free = torch.cuda.mem_get_info(0)[0]
    if free < need:
        pytest.skip("2^33 slots of 4 bytes, a 4 GB record pool and the model need about %.0f GB free, %.1f GB are" % (need / 1e9, free / 1e9))
    lib = _lib.load()
    n_bases = 200_000_000
    text = torch.empty(lib.jfgpu_synth_fasta_bytes(n_bases) + 256, dtype=torch.uint8, device="cuda")
    try:
        n_text = _synth(lib, text, n_bases, 0x5EED2048 + mode)
        queries = _queries(text, K, n_bases)
        model = km.count(text[:n_text], K, queries=queries)
        torch.cuda.empty_cache()
        with HashCounter(1 << 33, 7, k=K, canonical=True, region_mb=128, pool_bytes=4 << 30, k2_mode=mode) as hc:
            info = hc.info()
            assert (info["lsize"], info["slot_bits"], info["part_regions"], info["part_rec_bytes"]) == (33, 32, 256, 4), info
            hc.clear()
            hc.add_device_text(text.data_ptr(), n_text)
            st = hc.done()
            what = "2048 windows per region, k2_mode %d" % mode
            _check_step(hc, st, text[:n_text], K, info, model, queries, what)
            _check_dump(hc, text[:n_text], K, info, model, what + ", dump")
            assert st["seconds_win_scatter"] > 0 and st["seconds_win_insert"] > 0
            assert (st["seconds_win_hist"] > 0) == (mode == 4)
    finally:
        del text
        torch.cuda.empty_cache()
