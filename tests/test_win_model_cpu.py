"""The models of tests/win_model.py on hand-built cases, and the kernel harness tests/win_harness.cu compiled for sm_90a, so
that a change to the device structures it fills (WinDev, PartDev, TableDev) breaks this CPU test rather than a GPU session.
No GPU is needed."""
import collections
import os

import numpy as np
import pytest

import win_model as wm

def _pool(chunks):
    """A pool of the given record lists, one chunk each, in that order."""
    pool = np.zeros((len(chunks), wm.CHUNK_RECS), np.uint32)
    for c, recs in enumerate(chunks):
        pool[c, :len(recs)] = recs
    return pool, np.array([len(r) for r in chunks], np.uint32)


def test_placement_of_a_window_at_exactly_cap():
    """wpr 4, hb 10: window 2 of region 1 gets exactly cap = 8 records over two chunks, one chunk's stale tail past its
    directory count is ignored, and the exact layout pads every run to 4 records."""
    hb, wpr_lg = 10, 2
    rec = lambda w, x: (((w << wm.WIN_LG) | x) << hb) | (x & 0x3FF)
    region0 = [rec(0, 1), rec(3, 2), rec(3, 3)]
    hot = [rec(2, i) for i in range(8)]
    pool, dir_n = _pool([region0, hot[:5], hot[5:] + [rec(1, 7)]])
    pool[0, 3] = rec(1, 99)                                   # past dir_n[0]: not a record
    order = np.array([0, 2, 1], np.uint32)                    # region 0: chunk 0; region 1: chunks 2 and 1
    m = wm.place(pool, dir_n, order, [0, 1, 3], wpr_lg, hb)
    assert m.counts.tolist() == [1, 0, 0, 2, 0, 1, 8, 0]
    assert not m.overflows(8) and m.overflows(7)
    assert m.window(6).tolist() == sorted(hot)
    assert m.exact.tolist() == [0, 4, 4, 4, 8, 8, 12, 20, 20]
    # runs read back from a bucket layout are the same multisets, whatever order they were stored in
    cap = 8
    wrec = np.full(8 * cap, 0xFFFFFFFF, np.uint32)
    for i in range(8):
        wrec[i * cap:i * cap + m.counts[i]] = m.window(i)[::-1]
    got = wm.runs_of(wrec, np.arange(9) * cap, m.counts)
    assert wm.first_difference(m, got) is None
    wrec[6 * cap + 7] ^= 1
    assert "window 6" in wm.first_difference(m, wm.runs_of(wrec, np.arange(9) * cap, m.counts))


def test_a_probe_that_leaves_its_window():
    """Two keys at the last slot of window 0: the second takes probe 1, the first slot of window 1; decoding gives both
    their original position back."""
    t = wm.Table32(16, 13, 7)
    assert t.add(wm.WIN_SLOTS - 1, 5) == (wm.WIN_SLOTS - 1, True)
    assert t.add(wm.WIN_SLOTS - 1, 6) == (wm.WIN_SLOTS, True)
    assert t.add(wm.WIN_SLOTS - 1, 6) == (wm.WIN_SLOTS, False)
    t.add(wm.WIN_SLOTS - 1, 7)                                # probe 2: slot + 3
    d = wm.decode(t.slots, t.fbits, t.rbits, t.max_reprobe)
    assert d.as_dict() == {(wm.WIN_SLOTS - 1, 5): 1, (wm.WIN_SLOTS - 1, 6): 2, (wm.WIN_SLOTS - 1, 7): 1}
    assert sorted(zip(d.slot.tolist(), d.probe.tolist())) == [(wm.WIN_SLOTS - 1, 0), (wm.WIN_SLOTS, 1), (wm.WIN_SLOTS + 2, 2)]
    # the last slot of the table: probes go into the margin, not around
    t.add(t.local_size - 1, 1)
    assert t.add(t.local_size - 1, 2) == (t.local_size, True)


def test_counter_carries_and_the_side_table():
    """fbits 22 leaves a 10-bit counter: 2500 occurrences are 2 carries and 452 in the slot, and the side table in the
    device's layout decodes to the same count."""
    t = wm.Table32(15, 22, 7)
    s, new = t.add(1234, 77, 1000)
    t.add(1234, 77, 1500)
    assert new and t.carries == {s: 2} and int(t.slots[s]) >> 22 == 452
    keys, vals = t.ovf_arrays(1024)
    assert wm.carries_of(keys, vals) == {s: 2}
    assert wm.decode(t.slots, 22, 7, 126, wm.carries_of(keys, vals)).as_dict() == {(1234, 77): 2500}


def test_decoding_does_not_depend_on_insertion_order():
    """The same multiset of records inserted in two shuffled orders fills different slots but decodes to the same map,
    the model's count of every key; the judge accepts either table and rejects each kind of damage."""
    rng = np.random.default_rng(7)
    fb, rb = 20, 7
    pos = np.concatenate([rng.integers(16000, 16384, 3000),   # crowded: long chains, many leave window 0
                          30000 + 100 * np.arange(20)])       # and a few keys alone
    high = rng.integers(0, 1 << (fb - rb), len(pos)) & 7
    want = collections.Counter(zip(pos.tolist(), high.tolist()))
    tables = []
    for seed in (1, 2):
        t = wm.Table32(16, fb, rb)
        for j in np.random.default_rng(seed).permutation(len(pos)):
            t.add(int(pos[j]), int(high[j]))
        tables.append(t)
    assert not np.array_equal(tables[0].slots, tables[1].slots)
    empty = wm.decode(np.zeros(10, np.uint32), fb, rb, 126)
    for t in tables:
        d = wm.decode(t.slots, fb, rb, 126)
        assert d.as_dict() == dict(want)
        touched = np.zeros(len(t.slots), bool)
        touched[:2 * wm.WIN_SLOTS] = True
        before = np.zeros_like(t.slots)
        wm.judge(t.slots, d, before, wm.expected_map(empty, pos, high), touched, zero_windows=[3])
    t = tables[0]
    d = wm.decode(t.slots, fb, rb, 126)
    touched = np.ones(len(t.slots), bool)
    want_map = wm.expected_map(empty, pos, high)
    far = int(d.slot[np.argmax(d.probe)])                     # a hole in a probe chain
    bad = t.slots.copy()
    bad[int(d.pos[np.argmax(d.probe)])] = 0
    with pytest.raises(AssertionError, match="is empty|keys, the model"):
        wm.judge(bad, wm.decode(bad, fb, rb, 126), t.slots, want_map, touched)
    bad = t.slots.copy()                                      # a key twice: a probe-0 key copied to its empty probe 1
    s0 = next(int(s) for s, i in zip(d.slot, d.probe) if i == 0 and t.slots[s + 1] == 0)
    bad[s0 + 1] = (bad[s0] & ~np.uint32((1 << rb) - 1)) | np.uint32(2)
    with pytest.raises(AssertionError, match="in slots"):
        wm.judge(bad, wm.decode(bad, fb, rb, 126), t.slots, want_map, touched)
    bad = t.slots.copy()                                      # a count off by one
    bad[far] += np.uint32(1 << fb)
    with pytest.raises(AssertionError, match="wrong counts"):
        wm.judge(bad, wm.decode(bad, fb, rb, 126), t.slots, want_map, touched)
    with pytest.raises(AssertionError, match="window 0 got no record"):
        wm.judge(t.slots, d, np.zeros_like(t.slots), want_map, touched, zero_windows=[0])
    garbage = t.slots.copy()
    garbage[50000] = 0xDEADBEEF
    with pytest.raises(AssertionError):
        wm.judge(garbage, wm.decode(garbage, fb, rb, 126), t.slots, want_map, np.zeros(len(t.slots), bool))


@pytest.mark.skipif(wm.NVCC is None, reason="nvcc is not installed")
def test_harness_compiles(tmp_path):
    so = wm.build_harness(str(tmp_path))
    assert os.path.getsize(so) > 0
