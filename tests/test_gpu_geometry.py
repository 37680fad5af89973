"""A sweep of (k, table size) against plain Python models: the slot geometry of table_setup (jfutil.geometry), the counts
of a Counter of the text's k-mers and the (position, key) order of the dump.

The cases are chosen by rule: every k in 1..64 and lsize in 1..20 whose key field sits on either side of a slot-form
boundary (22/23: 32 -> 64 bits, 56/57: 64 -> 128, 64/65: the key field spills into the high word of a 128-bit slot,
120/121, and 127, the widest one), whose table is direct-indexed or nearly so (hb = 0 or 1), or that is requested larger
than the key space (lsize = 2k + 2, clipped to 4^k slots); and the wide form (k = 65, 96, 128) at a few sizes.  Every
text holds a poly-A stretch whose count carries out of the 32- and 64-bit forms' counters."""
import os
import random
import subprocess
from collections import Counter

import pytest

import jfutil
from jfutil import geometry

BOUNDARIES = (22, 23, 56, 57, 64, 65, 120, 121, 127)
POLY_A = 3000


def _select():
    cases = []
    for k in range(1, 65):
        for lsize in range(1, 21):
            g = geometry(k, lsize)
            if g["slot_bits"] and (g["fb"] in BOUNDARIES or g["hb"] in (0, 1) or lsize == 2 * k + 2):
                cases.append((k, lsize))
    return cases + [(k, lsize) for k in (65, 96, 128) for lsize in (1, 2, 3, 8, 16)]


CASES = _select()


def test_cases_cover_every_slot_form_and_both_sides_of_each_boundary():
    geo = [geometry(k, lsize) for k, lsize in CASES]
    assert len([g for g in geo if g["k"] <= 64]) == 188
    assert {(g["kw"], g["slot_bits"]) for g in geo} == {(1, 32), (1, 64), (1, 128), (2, 64), (2, 128), (4, 320)}
    fbs = {g["fb"] for g in geo if g["kw"] < 4}
    assert set(BOUNDARIES) <= fbs
    # the slot width changes across each boundary, and the 128-bit counter field shrinks to 1 bit at fb = 127
    widths = {g["fb"]: g["slot_bits"] for g in geo if g["kw"] < 4}
    assert (widths[22], widths[23], widths[56], widths[57], widths[121], widths[127]) == (32, 64, 64, 128, 128, 128)
    assert {g["cb"] for g in geo if g["kw"] < 4 and g["fb"] == 127} == {1}
    assert {g["cb"] for g in geo if g["kw"] < 4 and g["fb"] == 64} == {64}
    assert {g["cb"] for g in geo if g["kw"] < 4 and g["fb"] == 65} == {63}


def test_geometry_model_rejects_only_k64_at_eight_slots_or_fewer():
    rejected = [(k, lsize) for k in range(1, 129) for lsize in range(1, 21) if geometry(k, lsize)["slot_bits"] is None]
    assert rejected == [(64, 1), (64, 2), (64, 3)]


def _text(k, size, canonical, seed):
    """-> (FASTA bytes, the k-mers of the text in input order, keys of the text).  One record per k-mer, each key 1 to 3
    times, at most min(size/4, 4096) distinct keys with the poly-A one, so that the table never doubles."""
    rng = random.Random(seed)
    want = max(1, min(size // 4, 4096)) - 1
    seen, keys = {0}, []
    for _ in range(20 * want + 20):
        if len(keys) == want:
            break
        v = rng.getrandbits(2 * k)
        c = jfutil_canonical(v, k) if canonical else v
        if c not in seen:
            seen.add(c)
            keys.append(v)
    mers = []
    for i, v in enumerate(keys):
        mers += [v] * (1 + i % 3)
    rng.shuffle(mers)
    recs = [b">r\n" + int_to_mer(v, k).encode() + b"\n" for v in mers] + [b">a\n" + b"A" * POLY_A + b"\n"]
    return b"".join(recs), mers + [0] * (POLY_A - k + 1), keys + [0]


def jfutil_canonical(v, k):
    from jellyfish_b200.engine import canonical_int
    return canonical_int(v, k)


def int_to_mer(v, k):
    from jellyfish_b200.engine import int_to_mer
    return int_to_mer(v, k)


def _absent(k, canonical, present, n, seed):
    rng = random.Random(seed)
    out = []
    for _ in range(20 * n):
        if len(out) == n:
            break
        v = rng.getrandbits(2 * k)
        if (jfutil_canonical(v, k) if canonical else v) not in present:
            out.append(v)
    return out


@pytest.mark.gpu
def test_sweep_against_python_model(built):
    from jellyfish_b200 import HashCounter, reference_matrix
    for k, lsize in CASES:
        g = geometry(k, lsize)
        size, canonical = 1 << lsize, (k + lsize) % 2 == 0
        where = "k=%d lsize=%d canonical=%s" % (k, lsize, canonical)
        text, mers, keys = _text(k, 1 << g["lsize"], canonical, 1000 * k + lsize)
        norm = [jfutil_canonical(v, k) if canonical else v for v in mers]
        model = Counter(norm)
        with HashCounter(size, 7, k=k, canonical=canonical) as hc:
            hc.add_text(text)
            st = hc.done()
            info = hc.info()
            assert (info["lsize"], info["slot_bits"], info["max_reprobe"]) == (g["lsize"], g["slot_bits"], g["max_reprobe"]), where
            assert st["distinct"] == len(model), where
            if lsize < 2 * k:
                assert not info["matrix_identity"] and info["matrix_columns"] == reference_matrix(lsize, 2 * k), where
            else:
                assert info["matrix_identity"], where
            for ocl in (4, 8):
                assert hc.dump_records(out_counter_len=ocl) == jfutil.model_body(info, model, k, ocl), (where, ocl)
            absent = _absent(k, canonical, model, 100, lsize)
            assert hc.get_many(keys + absent) == [model[jfutil_canonical(v, k) if canonical else v] for v in keys] + [0] * len(absent), where
            for n in (3, 5000):
                want = [0] * n
                for c in model.values():
                    want[min(c, n - 1)] += 1
                assert hc.histogram(n) == want, (where, n)
            lines = b"".join(b"%s %d\n" % (int_to_mer(x, k).encode(), model[x]) for x in norm)
            assert hc.query_text(text) == lines, where
            body8 = jfutil.model_body(info, model, k, 8)
        with HashCounter(size, 7, k=k, canonical=canonical) as hc:
            hc.load_records(body8, 8)
            assert hc.dump_records(out_counter_len=8) == body8, where
        # three doublings smaller: the table grows back with later matrix draws, its final header orders the dump
        if lsize > 3 and geometry(k, lsize - 3)["slot_bits"]:
            with HashCounter(size >> 3, 7, k=k, canonical=canonical) as hc:
                hc.add_text(text)
                hc.done()
                info = hc.info()
                assert hc.dump_records() == jfutil.model_body(info, model, k, 4), where


@pytest.mark.gpu
def test_cli_rejects_k64_in_eight_slots(built, workdir, inputs):
    db = os.path.join(workdir, "k64_s8.jf")
    r = subprocess.run([jfutil.OUR_JF, "count", "-m", "64", "-s", "8", "-C", "-o", db, inputs["dangling.fa"]],
                       stdout=subprocess.PIPE, stderr=subprocess.PIPE)
    assert r.returncode != 0
    assert b"key too long for this table size (k=64, 8 slots" in r.stderr
    # one more slot doubling and it counts
    jfutil.run([jfutil.OUR_JF, "count", "-m", "64", "-s", "16", "-C", "-o", db, inputs["dangling.fa"]])
    assert jfutil.split_db(db)[0]["max_reprobe"] == 5
