"""Exact models of the window form of K2 (jellyfish_b200/csrc/jf_window.cuh), in numpy, for tests/test_gpu_win_kernels.py.

* `place`: what the bucket pass, win_scan and the exact pass must leave for one group: every window's records (as a sorted
  multiset) and count, whether some count exceeds the bucket capacity, and the exact layout (runs start on 16-byte
  boundaries: an exclusive scan of the counts rounded up to 4 records).
* `Table32`: sequential insertion into a table of 32-bit slots as large_hash_array does it: probe i of a key at position p
  is slot p + i(i+1)/2 (past the last slot into the margin, never around), its key field is (high << rbits) | (i + 1), the
  counter sits in the top 32 - fbits bits and a wrap adds one carry to the side table.
* `decode` and `judge`: a table (plus its carry side table) as {(original position, high): count}, and the checks a table
  filled by concurrent insertion must pass whatever order the records took.

A record of the window form is (position in region << hb) | high, 32 bits; its window in the region is
(record >> hb) >> WIN_LG.

`build_harness` compiles tests/win_harness.cu, the kernels behind a C ABI, with the library's flags."""
import os
import shutil
import subprocess

import numpy as np

WIN_LG = 14
WIN_SLOTS = 1 << WIN_LG
CHUNK_RECS = 2048                  # 4-byte records per 8 KB chunk
WIN_ST_UNITS = 12                  # chunks per tile of the bucket and exact passes
WIN2_RB = 10240                    # records per batch of win_insert2
WIN2_BLK = 256                     # records a consumer warp claims at a time
WIN_LAZY, WIN_IN_MEMORY = 0, 2
(STAT_KMERS, STAT_INSERTED, STAT_DISTINCT, STAT_REPROBES, STAT_OVERFLOWED, STAT_FAILED, STAT_FAIL_DROPPED, STAT_OVF_FULL,
 STAT_ROUTE_DROPPED, STAT_MAXCOUNT, STAT_POOL_FULL, STAT_FORMAT_ERR, STAT_N) = range(13)
GOLDEN = 0x9E3779B97F4A7C15
M64 = (1 << 64) - 1

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(os.path.dirname(HERE), "jellyfish_b200", "csrc")
NVCC = os.environ.get("NVCC") or shutil.which("nvcc") or next((p for p in ["/usr/local/cuda/bin/nvcc"] if os.path.exists(p)), None)
NVFLAGS = ["-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "--expt-relaxed-constexpr", "-Xcompiler", "-fPIC"]


def build_harness(out_dir):
    """Compile win_harness.cu into out_dir (the kernels from the engine's sources, in their own translation unit); returns
    the path of the shared library."""
    so = os.path.join(out_dir, "win_harness.so")
    r = subprocess.run([NVCC] + NVFLAGS + ["-shared", "-I", CSRC, "-o", so, os.path.join(HERE, "win_harness.cu")],
                       capture_output=True, text=True)
    if r.returncode:
        raise RuntimeError("nvcc failed:\n" + r.stdout + r.stderr)
    return so


def tri(i):
    return i * (i + 1) // 2


def round4(x):
    return (np.asarray(x, np.int64) + 3) & ~3


def bucket_cap(m, slack=True):
    """part_drain's bucket capacity for a largest mean of m records per window (k2_mode 4: no slack)."""
    c = m + int(np.ceil(6.0 * np.sqrt(m))) + 16 if slack else m
    return (c + 3) & ~3


# ---- placement -------------------------------------------------------------------------------------------------------
class Placement:
    """The records of one group by window: `counts` [n], `values` sorted by (window, value), `first` [n + 1] where each
    window's records start in `values`, and `exact` [n + 1], the run starts of the exact layout (exact[n] = its total)."""

    def __init__(self, tasks, values, n):
        o = np.lexsort((values, tasks))
        self.values = values[o].astype(np.uint32)
        self.counts = np.bincount(tasks, minlength=n).astype(np.int64)
        self.first = np.concatenate([[0], np.cumsum(self.counts)])
        self.exact = np.concatenate([[0], np.cumsum(round4(self.counts))])
        self.n = n

    def overflows(self, cap):
        return bool((self.counts > cap).any())

    def window(self, i):
        return self.values[self.first[i]:self.first[i + 1]]


def place(pool, dir_n, order, unit_first, wpr_lg, hb):
    """The model of one group: region r's records are the first min(dir_n[c], 2048) of every chunk c = order[u],
    u in [unit_first[r], unit_first[r + 1])."""
    G = len(unit_first) - 1
    tasks, values = [], []
    cols = np.arange(CHUNK_RECS)
    for r in range(G):
        units = np.asarray(order[unit_first[r]:unit_first[r + 1]], np.int64)
        if not len(units):
            continue
        n = np.minimum(np.asarray(dir_n, np.int64)[units], CHUNK_RECS)
        v = pool[units][cols[None, :] < n[:, None]]
        tasks.append((r << wpr_lg) + ((v >> np.uint32(hb + WIN_LG)) & np.uint32((1 << wpr_lg) - 1)).astype(np.int64))
        values.append(v)
    tasks = np.concatenate(tasks) if tasks else np.zeros(0, np.int64)
    values = np.concatenate(values) if values else np.zeros(0, np.uint32)
    return Placement(tasks, values, G << wpr_lg)


def runs_of(wrec, wstart, wcnt):
    """The records wstart/wcnt name in wrec, as a Placement (so each window's run is compared as a multiset)."""
    wcnt = np.asarray(wcnt, np.int64)
    n = len(wcnt)
    total = int(wcnt.sum())
    tasks = np.repeat(np.arange(n), wcnt)
    excl = np.concatenate([[0], np.cumsum(wcnt)[:-1]]) if n else np.zeros(0, np.int64)
    idx = np.repeat(np.asarray(wstart[:n], np.int64), wcnt) + (np.arange(total) - np.repeat(excl, wcnt))
    return Placement(tasks, np.asarray(wrec)[idx], n)


def first_difference(model, got):
    """None when every window holds the same multiset of records, else a description of the first window that does not."""
    bad = np.nonzero(model.counts != got.counts)[0]
    if len(bad):
        i = int(bad[0])
        return "window %d: %d records, the model has %d" % (i, got.counts[i], model.counts[i])
    diff = np.nonzero(model.values != got.values)[0]
    if len(diff):
        j = int(diff[0])
        i = int(np.searchsorted(model.first, j, side="right") - 1)
        return "window %d, record %d of its run: %#x, the model has %#x" % (i, j - model.first[i], got.values[j], model.values[j])
    return None


# ---- sequential insertion ----------------------------------------------------------------------------------------------
class Table32:
    """A table of 2^local_lsize 32-bit slots plus the margin of tri(max_reprobe) + 8 slots, filled one key at a time."""

    def __init__(self, local_lsize, fbits, rbits, max_reprobe=126):
        assert (max_reprobe + 1) >> rbits == 0 and fbits >= rbits
        self.local_lsize, self.fbits, self.rbits, self.max_reprobe = local_lsize, fbits, rbits, max_reprobe
        self.local_size = 1 << local_lsize
        self.slots = np.zeros(self.local_size + tri(max_reprobe) + 8, np.uint32)
        self.carries = {}                                 # slot -> carries (units of 2^(32 - fbits))

    def add(self, pos, high, count=1):
        """Add `count` to key (pos, high); returns (slot, whether the key is new).  Raises when no probe is free."""
        fb, rb = self.fbits, self.rbits
        fmask, cb = (1 << fb) - 1, 32 - fb
        assert 0 <= pos < self.local_size and 0 <= high < (1 << (fb - rb))
        for i in range(self.max_reprobe + 1):
            s = pos + tri(i)
            v = int(self.slots[s])
            kf = (high << rb) | (i + 1)
            if v == 0 or (v & fmask) == kf:
                c = (v >> fb) + count
                self.slots[s] = kf | ((c & ((1 << cb) - 1)) << fb)
                if c >> cb:
                    self.carries[s] = self.carries.get(s, 0) + (c >> cb)
                return s, v == 0
        raise RuntimeError("key (%d, %#x) found no slot in %d probes" % (pos, high, self.max_reprobe + 1))

    def ovf_arrays(self, size):
        """The carries as the device's side table (jf_device.cuh, ovf_add): tag slot + 1 at (slot * golden) >> 20, linear."""
        keys, vals = np.zeros(size, np.uint64), np.zeros(size, np.uint64)
        for s, c in sorted(self.carries.items()):
            h = ((s * GOLDEN) & M64) >> 20
            for i in range(4096):
                p = (h + i) & (size - 1)
                if keys[p] in (0, s + 1):
                    keys[p] = s + 1
                    vals[p] += c
                    break
            else:
                raise RuntimeError("side table full")
        return keys, vals


# ---- decoding and judging ----------------------------------------------------------------------------------------------
class Decoded:
    """The keys of a table: parallel arrays `slot`, `probe` (reprobe index), `pos` (original position), `high`, `count`,
    sorted by (pos, high)."""

    def __init__(self, slot, probe, pos, high, count, fbits, rbits):
        o = np.lexsort((high, pos))
        self.slot, self.probe, self.pos, self.high, self.count = slot[o], probe[o], pos[o], high[o], count[o]
        self.fbits, self.hbits = fbits, fbits - rbits

    @property
    def keys(self):
        return (self.pos.astype(np.uint64) << np.uint64(self.hbits)) | self.high.astype(np.uint64)

    def as_dict(self):
        return {(int(p), int(h)): int(c) for p, h, c in zip(self.pos, self.high, self.count)}


def carries_of(ovf_keys, ovf_vals):
    """slot -> carries of a side table."""
    nz = np.nonzero(ovf_keys)[0]
    return {int(ovf_keys[i]) - 1: int(ovf_vals[i]) for i in nz}


def decode(slots, fbits, rbits, max_reprobe, carries=None, skip=None):
    """Every nonzero slot s as a key: reprobe index i = (v & rmask) - 1, original position s - tri(i), high the bits between
    the reprobe field and the counter, count v >> fbits plus the carries of s.  `skip`: a boolean slot mask left out
    (windows whose memory is garbage by design).  Raises on a slot no insertion can have written."""
    slots = np.asarray(slots, np.uint32)
    s = np.nonzero(slots)[0]
    if skip is not None:
        s = s[~skip[s]]
    v = slots[s].astype(np.int64)
    i = (v & ((1 << rbits) - 1)) - 1
    bad = np.nonzero((i < 0) | (i > max_reprobe) | (s - i * (i + 1) // 2 < 0))[0]
    if len(bad):
        raise AssertionError("slot %d holds %#x: no key has that reprobe field" % (s[bad[0]], v[bad[0]]))
    hbits = fbits - rbits
    count = v >> fbits
    if carries:
        cs = np.array(sorted(carries), np.int64)
        at = np.minimum(np.searchsorted(s, cs), max(len(s) - 1, 0))
        hit = (s[at] == cs) if len(s) else np.zeros(len(cs), bool)
        add = np.zeros(len(s), np.int64)
        add[at[hit]] = [carries[int(x)] for x in cs[hit]]
        count = count + (add << (32 - fbits))
    return Decoded(s, i, s - i * (i + 1) // 2, (v >> rbits) & ((1 << hbits) - 1), count, fbits, rbits)


def expected_map(before, rec_pos, rec_high):
    """The counts a drain must leave: those of `before` (a Decoded) plus one per record (global position, high)."""
    want = before.as_dict()
    keys, counts = np.unique(np.stack([np.asarray(rec_pos, np.int64), np.asarray(rec_high, np.int64)]), axis=1, return_counts=True)
    for p, h, c in zip(keys[0].tolist(), keys[1].tolist(), counts.tolist()):
        want[p, h] = want.get((p, h), 0) + c
    return want


def judge(after, after_dec, before, want, touched, zero_windows=(), what=""):
    """Assert what a drain must leave, whatever the order its records were applied in:
    - no (position, high) twice;
    - every probe slot before a key's own slot occupied;
    - the map equals `want`;
    - a slot outside `touched` (a boolean slot mask: the windows that received records) unchanged, unless it holds a key of
      the map's records (a deferred record) which it held before or which took an empty slot;
    - the windows of `zero_windows` (window indices) all zero."""
    d = after_dec
    k = d.keys
    dup = np.nonzero(k[1:] == k[:-1])[0]
    assert not len(dup), "%s: key (%d, %#x) in slots %d and %d" % (what, d.pos[dup[0]], d.high[dup[0]], d.slot[dup[0]], d.slot[dup[0] + 1])
    for j in range(int(d.probe.max()) if len(d.probe) else 0):
        sel = np.nonzero(d.probe > j)[0]
        probe_slot = d.pos[sel] + j * (j + 1) // 2
        empty = np.nonzero(after[probe_slot] == 0)[0]
        assert not len(empty), "%s: key (%d, %#x) in slot %d (probe %d) but its probe %d, slot %d, is empty" % (
            what, d.pos[sel[empty[0]]], d.high[sel[empty[0]]], d.slot[sel[empty[0]]], d.probe[sel[empty[0]]], j, probe_slot[empty[0]])
    got = d.as_dict()
    if got != want:
        missing = sorted(set(want) - set(got))[:5]
        extra = sorted(set(got) - set(want))[:5]
        wrong = sorted(x for x in set(got) & set(want) if got[x] != want[x])[:5]
        raise AssertionError("%s: %d keys, the model has %d; missing %s; extra %s; wrong counts %s" % (
            what, len(got), len(want), missing, extra, [(x, got[x], want[x]) for x in wrong]))
    changed = np.nonzero((after != before) & ~touched)[0]
    if len(changed):
        ok = np.isin(changed, d.slot)
        assert ok.all(), "%s: slot %d outside the windows that got records changed from %#x to %#x" % (
            what, changed[~ok][0], before[changed[~ok][0]], after[changed[~ok][0]])
        fm = (1 << d.fbits) - 1                         # the key field: same key, or the slot was empty
        was = before[changed]
        assert ((was == 0) | ((was & np.uint32(fm)) == (after[changed] & np.uint32(fm)))).all(), \
            "%s: a deferred record overwrote another key outside its window" % what
    for w in zero_windows:
        seg = after[w * WIN_SLOTS:(w + 1) * WIN_SLOTS]
        nz = np.nonzero(seg)[0]
        assert not len(nz), "%s: window %d got no record in a write-only drain, but its slot %d holds %#x" % (what, w, nz[0], seg[nz[0]])
