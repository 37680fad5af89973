"""The window form of K2 (jf_window.cuh) kernel by kernel, launched through tests/win_harness.cu on inputs built to hit one
edge each, and judged by the exact models of tests/win_model.py.  A failure names the window and the record.

place   the bucket pass (K2b), win_scan and the exact pass (K2a) of one group: wcursor after the bucket pass, the flag,
        wstart, wcnt and every window's run (as a multiset) against the model, at 2 to 2048 windows per region, 1 to 64
        regions, 1 to 5 n_sm + 7 tiles, empty regions, chunk fills of 1..5, 2047 and 2048 records, and windows at exactly
        the bucket capacity and one past it.
insert  K2c (win_insert2), win_zero of a write-only drain and win_deferred: the decoded table against preloaded content plus
        the records, at windows of 0 to 30 725 records (batches of WIN2_RB, blocks of WIN2_BLK), CTA strides meeting 0..7
        windows, probes leaving the group and the table, counter carries, load 0.8, and lazy windows.

The harness compiles the kernels from the engine's sources in its own translation unit: it checks the source, while the
end-to-end tests judge the library's own build."""
import ctypes as C
import zlib

import numpy as np
import pytest

import win_model as wm

pytestmark = pytest.mark.gpu

FILL = 0xA5A5A5A5                          # wrec before the bucket pass
OVF_SIZE = 1 << 16
u32p = lambda a: C.c_void_p(a.ctypes.data)


class Harness:
    def __init__(self, so):
        self.lib = C.CDLL(so)
        v, u32, u64 = C.c_void_p, C.c_uint32, C.c_uint64
        self.lib.win_harness_n_sm.restype = C.c_int
        self.lib.win_harness_place.argtypes = [v, u32, v, v, u32, v, u32, u32, u32, u32, u32, u64, u32, u32,
                                               v, v, v, v, v, u64, v, C.c_char_p, C.c_size_t]
        self.lib.win_harness_insert.argtypes = [v, u32, u32, u32, u32, v, u32, u32, u32, v, v, v, u64, v, v, u64,
                                                v, v, C.c_char_p, C.c_size_t]
        self.n_sm = self.lib.win_harness_n_sm()
        assert self.n_sm > 0

    def place(self, g, cap, wrec_cap, flag0):
        n = g.G << g.wpr_lg
        out = dict(flag=np.zeros(1, np.uint32), wcursor=np.zeros(n, np.uint32), wstart=np.zeros(n + 1, np.uint32),
                   wcnt=np.zeros(n, np.uint32), wrec=np.zeros(wrec_cap, np.uint32), pool_full=np.zeros(1, np.uint64))
        err = C.create_string_buffer(512)
        rc = self.lib.win_harness_place(u32p(g.pool), len(g.pool), u32p(g.dir_n), u32p(g.order), len(g.order), u32p(g.unit_first),
                                        g.g0, g.G, g.wpr_lg, g.hb, cap, wrec_cap, flag0, FILL,
                                        u32p(out["flag"]), u32p(out["wcursor"]), u32p(out["wstart"]), u32p(out["wcnt"]),
                                        u32p(out["wrec"]), wrec_cap, u32p(out["pool_full"]), err, 512)
        assert rc == 0, err.value.decode()
        return out

    def insert(self, c, table, state, wstart, wcnt, wrec, ovf_keys, ovf_vals):
        stats, def_n = np.zeros(wm.STAT_N, np.uint64), np.zeros(1, np.uint64)
        err = C.create_string_buffer(512)
        rc = self.lib.win_harness_insert(u32p(table), c.local_lsize, c.fbits, c.rbits, c.max_reprobe,
                                         u32p(state) if state is not None else None, c.g0, c.G, c.wpr_lg,
                                         u32p(wstart), u32p(wcnt), u32p(wrec), len(wrec), u32p(ovf_keys), u32p(ovf_vals), len(ovf_keys),
                                         u32p(stats), u32p(def_n), err, 512)
        assert rc == 0, err.value.decode()
        return stats, int(def_n[0])


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    if wm.NVCC is None:
        pytest.skip("nvcc is not installed")
    return Harness(wm.build_harness(str(tmp_path_factory.mktemp("win_harness"))))


# ---- place: K2b + win_scan + K2a ---------------------------------------------------------------------------------------
class Group:
    """One group as part_drain hands it to the scatter passes.  `units`: per region, the record arrays of its units in
    order.  The chunks lie scattered over a pool with unused chunks between them, as K1's arenas leave them, and every
    chunk's tail past its directory count holds stale records."""

    def __init__(self, rng, units, g0, wpr_lg, hb):
        self.g0, self.G, self.wpr_lg, self.hb = g0, len(units), wpr_lg, hb
        flat = [u for r in units for u in r]
        n_chunks = len(flat) + 1 + len(flat) // 8
        self.pool = rng.integers(0, 1 << 32, (n_chunks, wm.CHUNK_RECS), dtype=np.uint32)
        self.dir_n = rng.integers(0, wm.CHUNK_RECS + 1, n_chunks).astype(np.uint32)
        self.order = rng.permutation(n_chunks)[:len(flat)].astype(np.uint32)
        for c, recs in zip(self.order, flat):
            self.pool[c, :len(recs)] = recs
            self.dir_n[c] = len(recs)
        self.unit_first = np.concatenate([[0], np.cumsum([len(r) for r in units])]).astype(np.uint32)
        self.tiles = [-(-len(r) // wm.WIN_ST_UNITS) for r in units]
        self.model = wm.place(self.pool, self.dir_n, self.order, self.unit_first, wpr_lg, hb)

    def m(self):
        """The largest mean of records per window over the regions (part_drain's m)."""
        per_region = self.model.counts.reshape(self.G, -1).sum(1)
        return int(-(-per_region.max() // (1 << self.wpr_lg)))


def records(rng, n, wpr_lg, hb, windows=None):
    """n records of a region: random positions (in `windows` when given) and random key bits below hb."""
    w = rng.integers(0, 1 << wpr_lg, n) if windows is None else np.asarray(windows)[rng.integers(0, len(windows), n)]
    pos = (w.astype(np.uint64) << np.uint64(wm.WIN_LG)) | rng.integers(0, wm.WIN_SLOTS, n).astype(np.uint64)
    return ((pos << np.uint64(hb)) | rng.integers(0, 1 << hb, n).astype(np.uint64)).astype(np.uint32)


FILLS = np.array([1, 2, 3, 4, 5, 2047, 2048])
FILL_P = np.array([1, 1, 1, 1, 1, 2, 8]) / 15.0


def check_place(h, g, cap, mode, wrec_cap=None):
    """Run the three kernels on group g and compare everything they return with the model."""
    cap = max(4, cap)
    m = g.model
    n = g.G << g.wpr_lg
    wrec_cap = wrec_cap or max(n * cap, int(m.exact[-1]))
    out = h.place(g, cap, wrec_cap, 1 if mode == 3 else 0)
    what = "wpr_lg %d, G %d, g0 %d, hb %d, tiles %s, cap %d, mode %d" % (g.wpr_lg, g.G, g.g0, g.hb, sum(g.tiles), cap, mode)
    bad = np.nonzero(out["wcursor"] != m.counts)[0]
    assert not len(bad), "%s: after the bucket pass wcursor[%d] = %d, the model counts %d" % (what, bad[0], out["wcursor"][bad[0]], m.counts[bad[0]])
    bad = np.nonzero(out["wcnt"] != m.counts)[0]
    assert not len(bad), "%s: wcnt[%d] = %d, the model counts %d" % (what, bad[0], out["wcnt"][bad[0]], m.counts[bad[0]])
    flagged = mode == 3 or m.overflows(cap)
    assert int(out["flag"][0]) == int(flagged), "%s: flag %d, largest window %d" % (what, out["flag"][0], m.counts.max())
    want = m.exact if flagged else np.arange(n + 1, dtype=np.int64) * cap
    bad = np.nonzero(out["wstart"] != want)[0]
    assert not len(bad), "%s: wstart[%d] = %d, expected %d" % (what, bad[0], out["wstart"][bad[0]], want[bad[0]])
    diff = wm.first_difference(m, wm.runs_of(out["wrec"], out["wstart"], out["wcnt"]))
    assert diff is None, "%s: %s" % (what, diff)
    assert int(out["pool_full"][0]) == 0, what
    return out, flagged


# (wpr_lg, G, g0, hb below the full width by, tiles of the group as (a, b): a * n_sm + b)
SWEEP = {
    "wpr2_G1_tile1": (1, 1, 0, 0, (0, 1)),
    "wpr4_G2_g0_7_lowhb": (2, 2, 7, 3, (1, -1)),
    "wpr32_G12_nsm": (5, 12, 40, 0, (1, 0)),
    "wpr512_G12_lowhb_nsm+1": (9, 12, 1, 2, (1, 1)),
    "wpr1024_G64_2nsm": (10, 64, 0, 0, (2, 0)),
    "wpr2048_G2_5nsm+7": (11, 2, 254, 0, (5, 7)),
    "wpr2048_G64_lowhb": (11, 64, 128, 3, (1, 1)),
}


def sweep_group(rng, n_sm, wpr_lg, G, g0, hb_low, tiles):
    """A group of `tiles` tiles over G regions; for G >= 3 the first, a middle and the last region are empty.  A region's
    chunk count is 0, 1 or 11 modulo 12 in turn; chunk fills are drawn from FILLS."""
    T = tiles[0] * n_sm + tiles[1]
    hb = 32 - wm.WIN_LG - wpr_lg - hb_low
    busy = [r for r in range(G) if G < 3 or r not in (0, G // 2, G - 1)]
    per = [0] * G
    for i in range(T):
        per[busy[i % len(busy)]] += 1
    units = []
    for i, r in enumerate(range(G)):
        nu = 0 if per[r] == 0 else wm.WIN_ST_UNITS * per[r] - (0, 11, 1)[i % 3]
        fills = rng.choice(FILLS, nu, p=FILL_P)
        units.append([records(rng, int(f), wpr_lg, hb) for f in fills])
    return Group(rng, units, g0, wpr_lg, hb)


@pytest.mark.parametrize("mode", [0, 3, 4])
@pytest.mark.parametrize("name", sorted(SWEEP))
def test_place_geometry(harness, name, mode):
    """Every dimension of the placement: windows per region, regions, tiles against n_sm, empty regions, chunk counts
    modulo 12, partial chunks, key bits below the full width; bucket layout (mode 0), flag preset (3), no slack (4)."""
    rng = np.random.default_rng(zlib.crc32(name.encode()) + mode)
    g = sweep_group(rng, harness.n_sm, *SWEEP[name])
    assert sum(g.tiles) == SWEEP[name][4][0] * harness.n_sm + SWEEP[name][4][1]
    cap = wm.bucket_cap(g.m(), slack=mode != 4)
    check_place(harness, g, cap, mode)


CAP = 2000


def hot_group(rng, n_sm, target, where):
    """Two regions of 32 windows: region 0 of 5 tiles, region 1 of 2 n_sm + 3 tiles (its last chunk count 11 mod 12).
    Window 9 of region 1 gets `target` records: over every chunk of the region ("spread"), only in tiles that are the
    first of their CTA ("first"), or all but one record spread and the last in the group's last tile ("last").  Every
    other window stays well below CAP."""
    wpr_lg, hb = 5, 32 - wm.WIN_LG - 5
    others = [w for w in range(32) if w != 9]
    units = [[records(rng, int(f), wpr_lg, hb) for f in rng.integers(1, 40, 5 * wm.WIN_ST_UNITS)]]
    nu = wm.WIN_ST_UNITS * (2 * n_sm + 3) - 1
    hot = np.zeros(nu, np.int64)
    if where == "spread":
        np.add.at(hot, np.arange(target) % nu, 1)
    elif where == "first":                              # group tiles 5 .. n_sm - 1 = region 1's tiles 0 .. n_sm - 6
        first = wm.WIN_ST_UNITS * (n_sm - 5)
        np.add.at(hot, np.arange(target) % first, 1)
    else:
        last = wm.WIN_ST_UNITS * (2 * n_sm + 2)         # the first unit of the last tile
        np.add.at(hot, np.arange(target - 1) % last, 1)
        hot[nu - 1] += 1
    region1 = []
    for u in range(nu):
        recs = np.concatenate([records(rng, int(hot[u]), wpr_lg, hb, [9]), records(rng, int(rng.integers(0, 28)), wpr_lg, hb, others)])
        region1.append(rng.permutation(recs) if len(recs) else records(rng, 1, wpr_lg, hb, others))
    units.append(region1)
    return Group(rng, units, 3, wpr_lg, hb)


@pytest.mark.parametrize("where", ["spread", "first", "last"])
@pytest.mark.parametrize("extra", [0, 1])
def test_place_bucket_edge(harness, extra, where):
    """A window of exactly CAP records leaves the flag clear and its bucket full; one more sets the flag, and the exact pass
    places the group.  Its records come from tiles of many CTAs, so the overflow is crossed by whichever claim comes last."""
    rng = np.random.default_rng(100 + 10 * extra + len(where))
    g = hot_group(rng, harness.n_sm, CAP + extra, where)
    hot = (1 << g.wpr_lg) + 9
    assert g.model.counts[hot] == CAP + extra
    assert np.delete(g.model.counts, hot).max() < CAP - 200
    out, flagged = check_place(harness, g, CAP, 0)
    assert flagged == bool(extra)
    if not extra:                                       # the bucket is full to its last record
        assert sorted(out["wrec"][hot * CAP:(hot + 1) * CAP].tolist()) == g.model.window(hot).tolist()


@pytest.mark.parametrize("cap,mode", [(24576, 0), (24572, 0), (24576, 3)])
def test_place_whole_tile_in_one_window(harness, cap, mode):
    """A tile of 12 full chunks all in window 5: a run of 24 576 records, the largest rank the packed ranks hold.  With
    cap = 24 576 it fills its bucket exactly; 4 less and the group overflows."""
    rng = np.random.default_rng(cap + mode)
    wpr_lg, hb = 9, 32 - wm.WIN_LG - 9
    others = [w for w in range(1 << wpr_lg) if w != 5]
    tile = [records(rng, wm.CHUNK_RECS, wpr_lg, hb, [5]) for _ in range(wm.WIN_ST_UNITS)]
    rest = [records(rng, int(f), wpr_lg, hb, others) for f in rng.choice(FILLS, 3 * wm.WIN_ST_UNITS + 1, p=FILL_P)]
    g = Group(rng, [tile + rest, rest[:7]], 9, wpr_lg, hb)
    assert g.model.counts[5] == 24576 and np.delete(g.model.counts, 5).max() < 24572
    out, flagged = check_place(harness, g, cap, mode)
    assert flagged == (cap < 24576 or mode == 3)


# ---- insert: K2c + win_zero + win_deferred -----------------------------------------------------------------------------
class Drain:
    """A table of n_regions regions of 2^(WIN_LG + wpr_lg) slots, filled beforehand by the sequential model, and the records
    of one group [g0, g0 + G) by window (task = region of the group << wpr_lg | window)."""

    def __init__(self, wpr_lg, g0, G, n_regions, fbits=13, rbits=7, max_reprobe=126):
        self.wpr_lg, self.g0, self.G = wpr_lg, g0, G
        self.region_bits = wm.WIN_LG + wpr_lg
        self.local_lsize = self.region_bits + (n_regions - 1).bit_length()
        assert 1 << (self.local_lsize - self.region_bits) == n_regions
        self.fbits, self.rbits, self.max_reprobe = fbits, rbits, max_reprobe
        self.hb = fbits - rbits
        self.t = wm.Table32(self.local_lsize, fbits, rbits, max_reprobe)
        self.n = G << wpr_lg
        self.recs = {}                                  # task -> (local position, high)

    def base(self, task):
        return ((self.g0 + (task >> self.wpr_lg)) << self.region_bits) + ((task & ((1 << self.wpr_lg) - 1)) << wm.WIN_LG)

    def window_of(self, task):
        return self.base(task) >> wm.WIN_LG

    def add(self, task, local, high):
        a, b = self.recs.get(task, (np.zeros(0, np.int64), np.zeros(0, np.int64)))
        self.recs[task] = (np.concatenate([a, np.asarray(local, np.int64)]), np.concatenate([b, np.asarray(high, np.int64)]))

    def preload(self, rng, task_or_window, n_keys, global_window=False):
        """n_keys random keys of one window into the table (sequentially), each with a count of 1..3; returns them."""
        w = task_or_window if global_window else self.window_of(task_or_window)
        local = rng.integers(0, wm.WIN_SLOTS, n_keys)
        high = rng.integers(0, 1 << self.hb, n_keys)
        for x, y, c in zip(local.tolist(), high.tolist(), rng.integers(1, 4, n_keys).tolist()):
            self.t.add((w << wm.WIN_LG) + x, y, c)
        return local, high

    def layout(self, rng, kind):
        """wstart, wcnt, wrec: buckets of a common capacity (i * cap), or the exact layout (runs padded to 4 records);
        each window's records shuffled; the gaps hold stale records."""
        cnt = np.array([len(self.recs.get(i, ((),))[0]) for i in range(self.n)], np.int64)
        if kind == "bucket":
            cap = int(wm.round4(cnt.max())) + 4
            start = np.arange(self.n, dtype=np.int64) * cap
        else:
            start = np.concatenate([[0], np.cumsum(wm.round4(cnt))])[:-1]
        total = int(start[-1] + cnt[-1]) if self.n else 0
        wrec = rng.integers(0, 1 << 32, total + 3, dtype=np.uint32)
        wmask = (1 << self.wpr_lg) - 1
        for task, (local, high) in self.recs.items():
            rec = ((((task & wmask) << wm.WIN_LG) | local) << self.hb) | high
            wrec[start[task]:start[task] + len(rec)] = rng.permutation(rec.astype(np.uint64) & 0xFFFFFFFF).astype(np.uint32)
        return start.astype(np.uint32), cnt.astype(np.uint32), wrec

    def run(self, h, rng, kind, state=None, what=""):
        """One drain; judges the result and leaves it in self.t.  `state`: the window states of a write-only drain (the
        WIN_LAZY windows must already hold garbage).  Returns (statistics, deferred records)."""
        before = self.t.slots.copy()
        lazy = np.zeros(len(before), bool)
        if state is not None:
            for w in np.nonzero(state != wm.WIN_IN_MEMORY)[0]:
                lazy[w << wm.WIN_LG:(w + 1) << wm.WIN_LG] = True
        dec_before = wm.decode(before, self.fbits, self.rbits, self.max_reprobe, self.t.carries, skip=lazy)
        ovf_keys, ovf_vals = self.t.ovf_arrays(OVF_SIZE)
        wstart, wcnt, wrec = self.layout(rng, kind)
        table = before.copy()
        stats, def_n = h.insert(self, table, state, wstart, wcnt, wrec, ovf_keys, ovf_vals)
        carries = wm.carries_of(ovf_keys, ovf_vals)
        after = wm.decode(table, self.fbits, self.rbits, self.max_reprobe, carries)
        pos = np.concatenate([self.base(t) + l for t, (l, _) in sorted(self.recs.items())] or [np.zeros(0, np.int64)])
        high = np.concatenate([hh for _, (_, hh) in sorted(self.recs.items())] or [np.zeros(0, np.int64)])
        want = wm.expected_map(dec_before, pos, high)
        touched = lazy.copy()
        for task in self.recs:
            w = self.window_of(task)
            touched[w << wm.WIN_LG:(w + 1) << wm.WIN_LG] = True
        group = range(self.window_of(0), self.window_of(0) + self.n)
        zero = [w for w in group if state is not None and state[w] != wm.WIN_IN_MEMORY and (w - group[0]) not in self.recs]
        wm.judge(table, after, before, want, touched, zero, what)
        assert stats[wm.STAT_FAILED] == 0 and stats[wm.STAT_OVF_FULL] == 0 and stats[wm.STAT_POOL_FULL] == 0, (what, stats)
        assert stats[wm.STAT_INSERTED] == len(pos), (what, stats[wm.STAT_INSERTED], len(pos))
        assert stats[wm.STAT_DISTINCT] == len(want) - len(dec_before.pos), (what, stats[wm.STAT_DISTINCT], len(want) - len(dec_before.pos))
        self.t.slots[:] = table
        self.t.carries = carries
        self.recs = {}
        return stats, def_n


def random_records(rng, d, task, n, n_keys, from_keys=None):
    """n records of n_keys keys of window `task` (some of them `from_keys`, keys already in the table)."""
    local = rng.integers(0, wm.WIN_SLOTS, n_keys)
    high = rng.integers(0, 1 << d.hb, n_keys)
    if from_keys is not None and n_keys > 4:
        k = min(n_keys // 3, len(from_keys[0]))
        local[:k], high[:k] = from_keys[0][:k], from_keys[1][:k]
    pick = np.concatenate([np.arange(min(n, n_keys)), rng.integers(0, n_keys, max(0, n - n_keys))])
    d.add(task, local[pick], high[pick])


SIZES = [0, 1, 3, 255, 256, 257, 10239, 10240, 10241, 20480, 30725]


@pytest.mark.parametrize("kind", ["bucket", "exact"])
def test_insert_window_sizes(harness, kind):
    """One window of each size around WIN2_BLK and WIN2_RB, up to three batches, in a group of 16 windows (fewer than
    SMs: most CTAs get none); every window preloaded with 3000 keys, a third of each window's keys among them."""
    rng = np.random.default_rng(11 if kind == "bucket" else 12)
    d = Drain(4, 1, 1, 4)
    for task, n in enumerate(SIZES + [0] * (16 - len(SIZES))):
        pre = d.preload(rng, task, 3000)
        if n:
            random_records(rng, d, task, n, min(n, 5000), pre)
    stats, _ = d.run(harness, rng, kind, what="window sizes, %s layout" % kind)
    assert stats[wm.STAT_INSERTED] == sum(SIZES)


def test_insert_cta_strides(harness):
    """64 regions of 16 windows: CTA b's stride (windows b, b + n_sm, ...) holds 0, 1, 2, 3 or 7 non-empty windows in
    turn, with empty windows between them."""
    rng = np.random.default_rng(13)
    d = Drain(4, 0, 64, 64)
    n_sm = harness.n_sm
    for b in range(n_sm):
        mine = list(range(b, d.n, n_sm))
        k = (0, 1, 2, 3, 7)[b % 5]
        assert len(mine) >= k
        pick = mine[:7] if k == 7 else sorted(rng.choice(mine, k, replace=False).tolist())
        for task in pick:
            n = int(rng.integers(1, 700))
            random_records(rng, d, task, n, max(1, n // 2))
    d.run(harness, rng, "exact", what="CTA strides")


@pytest.mark.parametrize("at_end", [False, True])
def test_insert_deferred_past_the_group(harness, at_end):
    """Records at the last slots of the group's last window, whose tail is full: their probes leave the window and the
    deferred kernel places them in the next region (a group in the middle of the table) or in the margin past the table
    (the group at its end).  Some of them are keys the sequential model had already pushed out of the window."""
    rng = np.random.default_rng(14 + at_end)
    d = Drain(2, 5 if at_end else 2, 3, 8)
    last = d.n - 1
    base = d.base(last)
    for x in range(wm.WIN_SLOTS - 64, wm.WIN_SLOTS):   # the window's tail full, several keys pushed past its end
        for y in range(3):
            d.t.add(base + x, y)
    if not at_end:
        d.preload(rng, (base >> wm.WIN_LG) + 1, 2000, global_window=True)       # the next region's first window
    local = np.repeat(np.arange(wm.WIN_SLOTS - 40, wm.WIN_SLOTS), 6)
    high = np.tile(np.arange(6), 40)                     # keys 0..2 are in the table already, 3..5 are new
    d.add(last, local, high)
    for task in range(d.n - 1):
        random_records(rng, d, task, 500, 300)
    in_margin = np.count_nonzero(d.t.slots[d.t.local_size:])
    stats, def_n = d.run(harness, rng, "exact", what="deferred, group %s" % ("at the end" if at_end else "in the middle"))
    assert def_n >= 40 * 3                               # (the new keys at least: every slot of the tail is taken)
    if at_end:
        assert np.count_nonzero(d.t.slots[d.t.local_size:]) >= in_margin + 40 * 3


def test_insert_hot_key_carries(harness):
    """fbits 22 leaves a 10-bit counter.  Window 0: a key preloaded at 1000 gets 25 000 more occurrences over three
    batches (25 carries in all); window 1: a new key gets 2049 (2 carries).  The side table holds exactly those."""
    rng = np.random.default_rng(15)
    d = Drain(1, 0, 1, 2, fbits=22)
    s_hot, _ = d.t.add(700, 0x55, 1000)
    d.preload(rng, 0, 2000)
    d.add(0, np.full(25000, 700), np.full(25000, 0x55))
    random_records(rng, d, 0, 5000, 2000)
    d.add(1, np.full(2049, 9), np.full(2049, 0x1ABC))
    random_records(rng, d, 1, 300, 100)
    d.run(harness, rng, "bucket", what="hot keys")
    assert d.t.carries.get(s_hot) == 26000 // 1024
    s2 = next(s for s in d.t.carries if s != s_hot)
    assert d.t.carries[s2] == 2 and d.t.slots[s2] >> 22 == 1


def test_insert_load_0_8(harness):
    """A window at load 0.8: 8192 keys preloaded, 4915 new keys in 15 000 records; long probe chains, no failure."""
    rng = np.random.default_rng(16)
    d = Drain(1, 0, 1, 2)
    pre = d.preload(rng, 0, 8192)
    random_records(rng, d, 0, 15000, 3 * 4915 // 2, pre)   # a third of the keys preloaded, 4915 new
    d.run(harness, rng, "exact", what="load 0.8")
    dec = wm.decode(d.t.slots, d.fbits, d.rbits, d.max_reprobe)
    assert (dec.pos < wm.WIN_SLOTS).sum() >= 0.79 * wm.WIN_SLOTS and dec.probe.max() >= 20


def test_insert_lazy_drain_then_a_second_drain(harness):
    """A write-only drain: of the group's 16 windows, WIN_LAZY ones hold 0xDEADBEEF and receive records or not, WIN_IN_MEMORY
    ones are preloaded and receive records or not.  The lazy windows that get no record must come out zero, the others
    hold exactly their records; then a second drain, not lazy, into the result."""
    rng = np.random.default_rng(17)
    d = Drain(3, 1, 2, 4)
    state = np.full(d.t.local_size >> wm.WIN_LG, wm.WIN_IN_MEMORY, np.uint32)
    for w in range(d.t.local_size >> wm.WIN_LG):
        if not d.window_of(0) <= w < d.window_of(0) + d.n:
            d.preload(rng, w, 1500, global_window=True)
    kinds = {}
    for task in range(d.n):
        lazy, gets = task % 4 in (0, 1), task % 2 == 0
        kinds[task] = (lazy, gets)
        w = d.window_of(task)
        pre = None
        if lazy:
            state[w] = wm.WIN_LAZY
        else:
            pre = d.preload(rng, task, 4000)
        if gets:
            random_records(rng, d, task, 6000 + 1000 * task, 3000, pre)
    for w in np.nonzero(state == wm.WIN_LAZY)[0]:
        d.t.slots[w << wm.WIN_LG:(w + 1) << wm.WIN_LG] = 0xDEADBEEF
    d.run(harness, rng, "exact", state=state, what="write-only drain")
    for task in range(d.n):
        random_records(rng, d, task, 2000, 1500)
    d.run(harness, rng, "bucket", what="second drain")
