"""Pin the doubling cases of regrow_cases.py without a GPU: the geometry each one claims, the distinct-key count that makes a
case forced-size, and (when oracle/_ref has been built) that the C restatement ends at the same size and matrix when the
records of every input file are permuted."""
import os
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

import jfutil
import regrow_cases as R
import text_model

FORCED = [c["name"] for c in R.CASES if c["final_l"] is not None]
ORACLE_CASES = [n for n in FORCED if R.BY_NAME[n]["kind"] != "load"] + ["load_s64"]


def _claims_hold(g, claim, where):
    got = dict(slot_bits=g["slot_bits"], P=g["P"], rec_bytes=g["rec_bytes"], window=g["window"], lsize=g["lsize"])
    assert {x: got[x] for x in claim} == claim, where


@pytest.mark.parametrize("name", [c["name"] for c in R.CASES])
def test_geometry_claims(name):
    c = R.BY_NAME[name]
    g0 = R.part_geometry(c["k"], c["start_l"], c["reprobes"])
    _claims_hold(g0, c["start"], (name, "start"))
    carried = g0["max_reprobe"]
    if c["final_l"] is not None:
        assert c["reprobes"] == 126
        _claims_hold(R.part_geometry(c["k"], c["final_l"], carried), c["end"], (name, "end"))
    for i, claim in enumerate(c["extra"].get("after_pass", [])):
        _claims_hold(R.part_geometry(c["k"], claim["lsize"], carried), claim, (name, "after pass", i))


def test_geometry_rows_of_the_doubling_table():
    """The slot form, counter width, record size and insertion form on both sides of each doubling the cases cross."""
    g = R.part_geometry
    assert (g(17, 18)["slot_bits"], g(17, 18)["cb"], g(17, 19)["slot_bits"], g(17, 19)["cb"]) == (64, 41, 32, 10)
    assert (g(33, 16)["slot_bits"], g(33, 16)["cb"], g(33, 17)["slot_bits"], g(33, 17)["cb"]) == (128, 64, 64, 8)
    assert (g(14, 17)["P"], g(14, 18)["P"], g(14, 18)["rec_bytes"]) == (0, 256, 4)
    assert (g(17, 22)["region_bits"], g(17, 22)["window"], g(17, 23)["region_bits"], g(17, 23)["window"]) == (14, False, 15, True)
    a, b = g(12, 23), g(12, 24)
    assert (a["hb"], a["max_reprobe"], a["window"]) == (1, 126, True) and (b["hb"], b["max_reprobe"], b["window"]) == (0, 0, True)
    c = g(21, 3)
    assert c["max_reprobe"] == 3 and g(21, 18, c["max_reprobe"])["max_reprobe"] == 3 and g(21, 18, c["max_reprobe"])["P"] == 256
    assert g(40, 16)["rec_bytes"] == 16 and g(40, 20)["slot_bits"] == 128


def _sym(files):
    return text_model.stream([R.file_bytes(f) for f in files])


def distinct_keys(case):
    """-> (fewest, most) keys that end up in the table of a case, its largest count and its keys counted more than 127
    times (None, None for a load)."""
    k, can = case["k"], case["canonical"]
    if case["kind"] == "load":
        n = len(R.load_body()[1])
        return n, n, None, None
    keys, cnt, _ = text_model.counts(_sym(R.text_files(case)), k, can)
    top, hot = int(cnt.max()), int((cnt > 127).sum())
    if case["kind"] == "if":
        n = len(text_model.counts(_sym(case["passes"][0]), k, can)[0])
        return n, n, top, hot
    if case["kind"] == "bloom":
        # every key seen twice passes the filter; of the singletons, about bf_fp
        single = int((cnt == 1).sum())
        return len(keys) - single, len(keys) - single + 3 * case["extra"]["bf_fp"] * single, top, hot
    return len(keys), len(keys), top, hot


@pytest.mark.parametrize("name", FORCED)
def test_forced_size_bounds(name):
    c = R.BY_NAME[name]
    L = c["final_l"]
    lo, hi, top, hot = distinct_keys(c)
    assert lo > 1 << (L - 1), (name, lo)
    assert hi <= 0.7 * (1 << L) or L == 2 * c["k"], (name, hi)
    if L == 2 * c["k"]:
        assert top < 1 << 7            # direct-indexed val_len growth is a known divergence (DESIGN.md section 7a)
    if hot is not None:
        assert hot <= 40, (name, hot)


def _oracle(case, files, out):
    args = R.oracle_args(case)
    if case["kind"] == "if":
        args += ["--if", files[0]]
        files = files[1:]
    jfutil.run([jfutil.ORACLE_C, "count"] + args + ["-o", out] + files)
    h, _ = jfutil.split_db(out)
    return h["size"], h["matrix1"]


@pytest.mark.skipif(not os.path.exists(jfutil.ORACLE_C), reason="oracle/_ref has not been built")
def test_restatement_size_does_not_depend_on_record_order(tmp_path):
    """Every forced-size case: the restatement ends at 2^L with the same matrix on the input and on two copies whose FASTA
    records are permuted (the k-mer multiset is the same).  The load case takes the matrix of a text with as many keys."""
    jobs = []
    for name in ORACLE_CASES:
        c = R.BY_NAME[name]
        names = ["load_text"] if c["kind"] == "load" else R.text_files(c)
        for perm in (None, 1, 2):
            paths = R.write_files(str(tmp_path), sorted(set(names)), perm)
            jobs.append((name, perm, [paths[f] for f in names], str(tmp_path / ("%s_%s.jf" % (name, perm)))))
    with ThreadPoolExecutor(max(1, min(8, os.cpu_count() or 1))) as ex:
        res = list(ex.map(lambda j: _oracle(R.BY_NAME[j[0]], j[2], j[3]), jobs))
    got = {}
    for (name, perm, _, _), (size, matrix) in zip(jobs, res):
        got.setdefault(name, []).append((size, matrix))
    for name, r in got.items():
        assert r[0][0] == 1 << R.BY_NAME[name]["final_l"], name
        assert r[1] == r[0] and r[2] == r[0], name
