"""Crafted counts at every counter boundary of every slot form, against plain Python integers.

A slot keeps the low cb bits of a count; the carries out of that field go to a side table and slot_full_count rebuilds
the count, saturating at 2^64 - 1.  Each form gets the counts 0, 1, around 2^cb and 2^(cb+1), around 2^32 and 2^56, 2^63
and the top of the 64-bit range, each on its own random key, loaded twice from a database body (so the model is
min(2c, 2^64 - 1)).  Then every reader of the table: lookup, histogram, the dump at every counter length and count
filter, query of a text and the CLI's `query -s` on the dumped database; the same after a load into 64 slots that has to
double several times (the counts move through collect_kernel).  Then the increment of one that carries out of a full
counter field, through every insertion path of the form."""
import os
import random

import pytest

import jfutil
from jfutil import geometry

TOP = (1 << 64) - 1

# name -> (k, lsize, key words, slot bits, in-slot counter bits)
FORMS = {
    "kw1_s32":       (12, 16, 1, 32, 17),
    "kw1_s64":       (21, 16, 1, 64, 31),
    "kw2_s64":       (33, 20, 2, 64, 11),
    "kw1_s128_cb64": (32, 14, 1, 128, 64),
    "kw2_s128_cb64": (33, 10, 2, 128, 64),
    "kw2_s128":      (63, 20, 2, 128, 15),
    "kw2_s128_cb7":  (64, 14, 2, 128, 7),
    "kw4_wide":      (100, 12, 4, 320, 56),
}
FILLER = 300          # keys with small counts beside the crafted ones (64 slots then double at least three times)


def boundary_counts(cb):
    c = [0, 1, (1 << cb) - 1, 1 << cb, (1 << cb) + 1, (1 << (cb + 1)) - 1, (1 << 32) - 1, 1 << 32, (1 << 56) - 1, 1 << 56,
         1 << 63, TOP - 1, TOP]
    return sorted(set(x for x in c if x <= TOP))


def _keys(k, n, seed):
    rng = random.Random(seed)
    out = []
    while len(out) < n:
        v = rng.getrandbits(2 * k)
        if v not in out:
            out.append(v)
    return out


def _body(k, pairs):
    kb = (2 * k + 7) // 8
    return b"".join(x.to_bytes(kb, "little") + c.to_bytes(8, "little") for x, c in pairs)


def _fasta(k, keys):
    from jellyfish_b200.engine import int_to_mer
    return b"".join(b">r%d\n%s\n" % (i, int_to_mer(x, k).encode()) for i, x in enumerate(keys))


def _lines(k, keys, model):
    from jellyfish_b200.engine import int_to_mer
    return b"".join(b"%s %d\n" % (int_to_mer(x, k).encode(), model[x]) for x in keys)


def test_forms_have_the_counter_widths_of_the_geometry_model():
    for name, (k, lsize, kw, sb, cb) in FORMS.items():
        g = geometry(k, lsize)
        assert (g["kw"], g["slot_bits"], g["cb"]) == (kw, sb, cb), name


def _check_readers(hc, k, model, crafted, cb, where):
    info = hc.info()
    assert hc.get_many(list(model)) == list(model.values()), where
    want = [0] * 16
    for c in model.values():
        want[min(c, 15)] += 1
    assert hc.histogram(16) == want, where
    for ocl in range(1, 9):
        assert hc.dump_records(out_counter_len=ocl) == jfutil.model_body(info, model, k, ocl), (where, ocl)
    for bound in sorted(set(b for b in (1 << cb, TOP) if b <= TOP)):
        assert hc.dump_records(lower=bound, out_counter_len=8) == jfutil.model_body(info, model, k, 8, lower=bound), (where, bound)
        assert hc.dump_records(upper=bound, out_counter_len=8) == jfutil.model_body(info, model, k, 8, upper=bound), (where, bound)
    assert hc.query_text(_fasta(k, crafted)) == _lines(k, crafted, model), where


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(FORMS))
def test_boundary_counts_through_every_reader(name, built, workdir):
    from jellyfish_b200 import HashCounter
    k, lsize, kw, sb, cb = FORMS[name]
    counts = boundary_counts(cb)
    keys = _keys(k, len(counts) + FILLER, sorted(FORMS).index(name) + 1)
    rng = random.Random(lsize)
    pairs = list(zip(keys, counts + [rng.randrange(1, 1000) for _ in range(FILLER)]))
    crafted = keys[:len(counts)]
    model = {x: min(2 * c, TOP) for x, c in pairs}
    first, second = _body(k, pairs), _body(k, pairs[::-1])
    assert any(len(str(c)) == 20 for c in model.values())
    with HashCounter(1 << lsize, 7, k=k) as hc:
        hc.load_records(first, 8)
        hc.load_records(second, 8)
        info = hc.info()
        assert (info["lsize"], info["slot_bits"]) == (lsize, sb)
        _check_readers(hc, k, model, crafted, cb, name)
        db = os.path.join(workdir, "counters_%s.jf" % name)
        hc.dump(db, out_counter_len=8)
    fa = os.path.join(workdir, "counters_%s.fa" % name)
    with open(fa, "wb") as f:
        f.write(_fasta(k, crafted))
    out = jfutil.run([jfutil.OUR_JF, "query", "-s", fa, db]).stdout
    assert out == _lines(k, crafted, model)
    # a table of 64 slots that doubles several times: collect_kernel moves the carried counts
    with HashCounter(64, 7, k=k) as hc:
        hc.load_records(first, 8)
        hc.load_records(second, 8)
        st = hc.done()
        assert st["regrows"] >= 3 and hc.info()["lsize"] >= 9
        _check_readers(hc, k, model, crafted, cb, name + " after doublings")


# the insertion paths of a count of one: (form, k, lsize, engine switches, check of the path taken)
WINDOW = dict(part_min_mb=1, pool_bytes=1 << 30, max_batch_bytes=1 << 20)
PATHS = [("direct_" + name, k, lsize, dict(no_partition=True)) for name, (k, lsize, _, _, _) in sorted(FORMS.items())]
for mode in (1, 2):
    PATHS += [("region%d_kw1_s32" % mode, 12, 18, dict(WINDOW, k2_mode=mode)),
              ("region%d_kw1_s64" % mode, 21, 17, dict(WINDOW, k2_mode=mode)),
              ("region%d_kw2_s64" % mode, 33, 20, dict(WINDOW, k2_mode=mode)),
              ("region%d_kw2_s128_cb64" % mode, 33, 16, dict(WINDOW, k2_mode=mode)),
              ("region%d_kw2_s128" % mode, 63, 20, dict(WINDOW, k2_mode=mode))]
PATHS += [("window%d_kw1_s32" % mode, 17, 23, dict(WINDOW, k2_mode=mode)) for mode in (0, 3)]


@pytest.mark.gpu
@pytest.mark.parametrize("path", PATHS, ids=[p[0] for p in PATHS])
def test_count_of_one_carries_out_of_a_full_counter(path, built):
    """Keys loaded at 2^cb - 1 and at 2^64 - 1, then fed once each as text: 2^cb (the one carry of table_add_batch,
    k2_settle / k2_walk, K2c's k2_carry and wide_count) and 2^64 - 1 (saturated)."""
    from jellyfish_b200 import HashCounter
    name, k, lsize, kw = path
    cb = geometry(k, lsize)["cb"]
    keys = _keys(k, 24, lsize * 131 + k)
    full, top = keys[:12], keys[12:]
    with HashCounter(1 << lsize, 7, k=k, **kw) as hc:
        info = hc.info()
        if name.startswith("direct"):
            assert info["part_regions"] == 0
        else:
            assert info["part_regions"] > 0
            if name.startswith("window"):
                assert info["slot_bits"] == 32 and info["part_rec_bytes"] == 4
        hc.load_records(_body(k, [(x, (1 << cb) - 1) for x in full] + [(x, TOP) for x in top]), 8)
        hc.add_text(_fasta(k, keys))
        st = hc.done()
        assert st["kmers"] == len(keys) and st["regrows"] == 0
        assert hc.get_many(keys) == [min(1 << cb, TOP)] * len(full) + [TOP] * len(top)
        model = {x: min(1 << cb, TOP) for x in full}
        model.update((x, TOP) for x in top)
        assert hc.dump_records(out_counter_len=8) == jfutil.model_body(hc.info(), model, k, 8)


@pytest.mark.gpu
def test_full_side_table_is_an_error(built):
    """k = 14 in 2^21 slots (32-bit slots, an 18-bit counter field, a side table of 2^20 entries): 1.2 M keys at 2^18 each
    need 1.2 M carry entries."""
    import numpy as np
    from jellyfish_b200 import HashCounter, JellyfishError
    from jellyfish_b200._lib import ERR_FULL
    k, lsize = 14, 21
    assert geometry(k, lsize)["cb"] == 18
    rng = np.random.default_rng(14)
    keys = np.unique(rng.integers(0, 1 << 28, size=1_400_000, dtype=np.uint64))
    keys = rng.permutation(keys)[:1_200_000]
    rec = np.zeros(len(keys), dtype=[("key", "<u4"), ("count", "<u8")])
    rec["key"] = keys.astype(np.uint32)
    rec["count"] = 1 << 18
    with HashCounter(1 << lsize, 7, k=k) as hc:
        with pytest.raises(JellyfishError) as ei:
            hc.load_records(rec.tobytes(), 8)
        assert ei.value.code == ERR_FULL and "counter overflow side table is full" in str(ei.value)
