"""Table doubling cases, shared by test_regrow_cases_cpu.py (no GPU) and test_gpu_regrow.py.

Every case starts a counter at a size it outgrows and names the geometry it claims at the start and at the end: slot bits,
regions of the record pool (`part_regions`), record bytes, and whether a drain at that size takes the window form of K2.
`part_geometry` restates `part_configure` (jellyfish_b200/csrc/jf_engine.cu) for those claims.

A case is *forced-size* (`final_l` set) when it keeps the default reprobe limit and its N distinct keys satisfy
2^(L-1) < N <= 0.7 * 2^L: fewer than N slots cannot hold the keys, and at a load of 0.7 no key needs 126 probes, so the
table ends at 2^L whatever the insertion order, and so do the reference and its C restatement (outside the 0.90-0.92 band
of DESIGN.md section 7a).  A table of 4^k slots (L = 2k) cannot fail at all and counts as forced too.  Only forced-size
cases are compared byte for byte with the restatement.  Hot keys (count > 127) stay a few dozen per case, so that the
reference's continuation entries cannot move its fill point.

Inputs are seeded: random FASTA in records of 300..3000 bases, plus hot records (one k-mer per record, repeated).  A pass
is a list of files fed before one `done()`; a path is a set of engine switches, with optional `passes_split`: the files of
each pass fed as that many passes."""
import functools
import math
import os
import random

import numpy as np

import jfutil

TOP = (1 << 64) - 1
WIN_LG, PMAX, RING_P, CHUNK_BYTES = 14, 2048, 1024, 8192         # jf_kernels.cuh, jf_extract.cuh
REGION = dict(part_min_mb=1, max_batch_bytes=1 << 20)


def tri(i):
    return i * (i + 1) // 2


def part_geometry(k, lsize, reprobe_limit=126, no_partition=False, part_min_mb=1, region_mb=64):
    """jfutil.geometry plus the record pool part_configure sets up for that table: P regions of 2^region_bits slots,
    rec_bytes per record (P = 0: direct insertion), and whether a drain takes the window form (window_enabled, k2_mode 0)."""
    g = dict(jfutil.geometry(k, lsize, reprobe_limit))
    g.update(P=0, region_bits=0, rec_bytes=0, window=False)
    sb, l, hb = g["slot_bits"], g["lsize"], g["hb"]
    margin = tri(g["max_reprobe"]) if g["max_reprobe"] else 0
    if g["kw"] == 4 or no_partition or ((1 << l) + margin + 8) * (sb // 8) < ((part_min_mb or 256) << 20):
        return g
    P = 256
    owned = (1 << l) * (sb // 8)
    while P < PMAX and owned // P > (region_mb << 20):
        P <<= 1
    lg = lambda x: x.bit_length() - 1
    if sb == 32 and l > lg(P):
        bits = l - lg(P) + hb
        extra = bits - 32 if bits > 32 else 0
        if extra and extra < 8 and (P << extra) <= RING_P and l - lg(P << extra) > WIN_LG:
            P <<= extra
    if P < 64 or l < 8 or (1 << (l - 8)) < P:
        return g
    region_bits = l - lg(P)
    bits = region_bits + hb
    rec = 4 if bits <= 32 else 8 if bits <= 64 else 16 if bits <= 128 else 0
    if not rec:
        return g
    mean = 1024.0 * 32 / P
    if int(mean + 6.0 * math.sqrt(mean) + 8.0) * 2 > CHUNK_BYTES // rec:
        return g
    g.update(P=P, region_bits=region_bits, rec_bytes=rec,
             window=sb == 32 and rec == 4 and WIN_LG < region_bits <= WIN_LG + 11)
    return g


# -- inputs ---------------------------------------------------------------------------------------------------------

def random_records(n, seed):
    """n random bases as FASTA records of 300..3000 bases (one k-mer window resets at every record)."""
    import gen
    seq = gen._seq(n, seed)
    rng = random.Random(seed ^ 0x5EED)
    out, i, r = [], 0, 0
    while i < n:
        ln = rng.randrange(300, 3001)
        out.append(b">r%d_%d\n%s\n" % (seed, r, seq[i:i + ln]))
        i += ln
        r += 1
    return out


def hot_records(k, counts, seed):
    """One random k-mer per count c, written as c records that hold only that k-mer: it is counted exactly c times."""
    import gen
    out = []
    for j, c in enumerate(counts):
        mer = gen._seq(k, seed * 1000 + j)
        out += [b">h%d\n%s\n" % (j, mer)] * c
    return out


def repeat_records(n, unit):
    """n bases of a periodic sequence (one record, 70-column lines)."""
    import gen
    return [gen.fasta((unit * (n // len(unit) + 1))[:n], name=b"rep")]


# name -> list of FASTA records (bytes each); a file is the concatenation of its records
FILES = {
    "k17_main":  lambda: random_records(4_600_000, 171) + hot_records(17, [1023, 1024, 2047, 2048, 16383, 16384], 171),
    "k17_more":  lambda: random_records(800_000, 172),
    "k33":       lambda: random_records(620_000, 331) + hot_records(33, [255, 256, 511, 512, 2047, 2048, 65535, 65536], 331),
    "k40":       lambda: random_records(620_000, 401) + hot_records(40, [127, 128, 255, 256, 4096], 401),
    "k14_a":     lambda: random_records(170_000, 141) + hot_records(14, [300, 1000], 141),
    "k14_b":     lambda: random_records(170_000, 142),
    "k12_a":     lambda: random_records(19_000_000, 121),
    "k12_b":     lambda: random_records(1_000_000, 122),
    "k21_grow":  lambda: random_records(300_000, 211) + hot_records(21, [200, 70000], 211),
    "k21_p10":   lambda: random_records(700_000, 212),
    "if_prime":  lambda: random_records(4_600_000, 181),
    "if_upd1":   lambda: random_records(4_600_000, 181)[::3] + random_records(500_000, 182) + hot_records(17, [130, 5000], 183),
    "if_upd2":   lambda: random_records(4_600_000, 181)[1::5] + random_records(300_000, 184),
    "spill":     lambda: random_records(1_000_000, 191) + repeat_records(30_000_000, b"ACG") + random_records(9_500_000, 192),
    "bf_a":      lambda: random_records(2_600_000, 221) + hot_records(21, [500], 221),
    "bf_b":      lambda: random_records(1_000_000, 222),
    "load_text": lambda: random_records(2_500_000, 231),
}


def file_bytes(name, permute_seed=None):
    recs = FILES[name]()
    if permute_seed is not None:
        recs = list(recs)
        random.Random(permute_seed).shuffle(recs)
    return b"".join(recs)


def write_files(d, names, permute_seed=None):
    """Write the named inputs under d (once) -> {name: path}."""
    out = {}
    for name in names:
        suffix = "" if permute_seed is None else "_perm%d" % permute_seed
        path = os.path.join(d, "regrow_%s%s.fa" % (name, suffix))
        if not os.path.exists(path):
            with open(path + ".tmp", "wb") as f:
                f.write(file_bytes(name, permute_seed))
            os.replace(path + ".tmp", path)
        out[name] = path
    return out


@functools.lru_cache(None)
def load_body(seed=71, n=2_500_000):
    """Case load_s64: n distinct random 21-mers as an 8-byte-count record body, with counts 1..1000 and the crafted counts
    2^31 + 5, 2^32 - 1, 2^32 and 2^63 -> (body, keys, counts), the last two uint64 arrays."""
    rng = np.random.default_rng(seed)
    keys = np.unique(rng.integers(0, 1 << 42, size=n + n // 50, dtype=np.uint64))
    keys = rng.permutation(keys)[:n]
    cnt = rng.integers(1, 1001, size=n).astype(np.uint64)
    crafted = [(1 << 32) - 1, 1 << 32, 1 << 63, (1 << 31) + 5]
    cnt[:len(crafted) * 3] = np.repeat(np.array(crafted, np.uint64), 3)
    rec = np.zeros(n, dtype=[("key", "<u8"), ("count", "<u8")])
    rec["key"], rec["count"] = keys, cnt
    raw = rec.view(np.uint8).reshape(n, 16)
    body = np.ascontiguousarray(np.concatenate((raw[:, :6], raw[:, 8:]), axis=1)).tobytes()      # 6 key bytes (42 bits)
    return body, keys, cnt


# -- the cases ------------------------------------------------------------------------------------------------------

def _case(name, k, canonical, start_l, passes, paths, start, end, final_l=None, reprobes=126, kind="count", extra=None):
    return dict(name=name, k=k, canonical=canonical, start_l=start_l, passes=passes, paths=paths, start=start, end=end,
                final_l=final_l, reprobes=reprobes, kind=kind, extra=extra or {})


def _claim(slot_bits, P, rec_bytes, window, lsize=None):
    d = dict(slot_bits=slot_bits, P=P, rec_bytes=rec_bytes, window=window)
    if lsize is not None:
        d["lsize"] = lsize
    return d


CASES = [
    # 1. 64-bit slots (41-bit counter) -> 32-bit slots (10-bit counter), five doublings inside one drain of the L2 form;
    # hot keys at 1023..4096 after the move.  Several drains: the same files in three passes, or a 64 MB pool.
    _case("s64_to_s32", 17, True, 18, [["k17_main"]],
          {"k2_1": dict(REGION, k2_mode=1), "k2_2": dict(REGION, k2_mode=2), "k2_1_pool64": dict(REGION, k2_mode=1, pool_bytes=64 << 20),
           "k2_2_passes3": dict(REGION, k2_mode=2, passes_split=3)},
          _claim(64, 256, 4, False), _claim(32, 256, 4, True), final_l=23),
    # 2. case 1, then a second feed into the table it grew: the first window-form drain of a rebuilt table
    _case("window_after_rebuild", 17, True, 18, [["k17_main"], ["k17_more"]],
          {"k2_0": dict(REGION, k2_mode=0), "k2_3": dict(REGION, k2_mode=3), "k2_4": dict(REGION, k2_mode=4)},
          _claim(64, 256, 4, False), _claim(32, 256, 4, True), final_l=23),
    # 3. two-word keys, 128-bit slots (64-bit counter, 8-byte records) -> 64-bit slots (8-bit counter), four doublings
    _case("s128_to_s64", 33, False, 16, [["k33"]],
          {"k2_1": dict(REGION, k2_mode=1), "k2_2": dict(REGION, k2_mode=2), "direct": dict(no_partition=True)},
          _claim(128, 256, 8, False), _claim(64, 256, 8, False), final_l=20),
    # 4. k = 40 stays on 128-bit slots and 16-byte records through four doublings (rehash_chunks_kernel<2, 128>)
    _case("s128_k40", 40, False, 16, [["k40"]],
          {"k2_2": dict(REGION, k2_mode=2), "k2_1": dict(REGION, k2_mode=1)},
          _claim(128, 256, 16, False), _claim(128, 256, 16, False), final_l=20),
    # 5. below the 1 MB floor (direct insertion) -> region records after the first doubling, then a region drain that doubles
    _case("direct_to_region", 14, True, 17, [["k14_a"], ["k14_b"]],
          {"k2_1": dict(REGION, k2_mode=1), "k2_2": dict(REGION, k2_mode=2)},
          _claim(32, 0, 0, False), _claim(32, 256, 4, False), final_l=19,
          extra=dict(after_pass=[_claim(32, 256, 4, False, lsize=18), _claim(32, 256, 4, False, lsize=19)])),
    # 6. hashed window form (hb = 1) -> 4^k slots: identity matrix, no reprobes, hb = 0; a second feed drains in that form
    _case("into_direct_index", 12, False, 23, [["k12_a"], ["k12_b"]],
          {"k2_0": dict(REGION, k2_mode=0, pool_bytes=1 << 30)},
          _claim(32, 256, 4, True), _claim(32, 256, 4, True), final_l=24),
    # 7. a record body loaded twice (stage_keys_kernel -> drain -> rehash), 64-bit slots and 8-byte records at the start
    _case("load_s64", 21, False, 18, [["@load"], ["@load_reversed"]],
          {"k2_1": dict(REGION, k2_mode=1), "direct": dict(no_partition=True)},
          _claim(64, 256, 8, False), _claim(64, 256, 8, False), final_l=22, kind="load"),
    # 8. --if: the PRIME drain doubles (L2 form, the rehash inserts count 0), UPDATE adds only to the primed keys
    _case("if_prime", 17, True, 18, [["if_prime"], ["if_upd1", "if_upd2"]],
          {"k2_1": dict(REGION, k2_mode=1), "direct": dict(no_partition=True)},
          _claim(64, 256, 4, False), _claim(32, 256, 4, True), final_l=23, kind="if"),
    # 9. a full spill list before the first drain (K1 inserts its overflow itself), a doubling mid-drain, then the spill list
    # into the doubled table
    _case("spill_then_double", 17, True, 23, [["spill"]],
          {"k2_0": dict(REGION, k2_mode=0, pool_bytes=1 << 30)},
          _claim(32, 256, 4, True), _claim(32, 256, 4, True), final_l=24),
    # 10. -s 8 clips the reprobe limit to 3 for good; the table grows far into region mode.  Order decides the final size:
    # own-geometry judges only.  Found here: rebuild_table (jf_engine.cu) counted a moved entry that found no slot in the new
    # table twice in STAT_INSERTED (once when it first landed, again when the next table took it from the failure list).
    _case("clipped_limit", 21, True, 3, [["k21_grow"]],
          {"direct": dict(no_partition=True), "k2_1": dict(REGION, k2_mode=1), "k2_2": dict(REGION, k2_mode=2)},
          _claim(64, 0, 0, False), None),
    _case("limit_p10", 21, True, 18, [["k21_p10"]],
          {"k2_1": dict(REGION, k2_mode=1), "k2_2": dict(REGION, k2_mode=2)},
          _claim(64, 256, 8, False), None, reprobes=10),
    # 11. Bloom prefilter in front of the region path: A twice, then B.  Forced-size with N = the keys that pass.
    _case("bloom_region", 21, True, 18, [["bf_a"], ["bf_a", "bf_b"]],
          {"k2_1": dict(REGION, k2_mode=1)},
          _claim(64, 256, 8, False), _claim(64, 256, 8, False), final_l=22, kind="bloom",
          extra=dict(bf_size=4_000_000, bf_fp=0.01)),
]
BY_NAME = {c["name"]: c for c in CASES}


def text_files(case):
    """The named FASTA inputs of a case, in feeding order."""
    return [f for p in case["passes"] for f in p if not f.startswith("@")]


def oracle_args(case):
    """jf_oracle count switches of a case (without -o and the input files)."""
    a = ["-m", str(case["k"]), "-s", str(1 << case["start_l"])]
    if case["canonical"]:
        a.append("-C")
    if case["reprobes"] != 126:
        a += ["-p", str(case["reprobes"])]
    if case["kind"] == "bloom":
        a += ["--bf-size", str(case["extra"]["bf_size"]), "--bf-fp", str(case["extra"]["bf_fp"])]
    return a
