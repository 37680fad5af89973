"""Table doubling on every insertion path, against exact models (cases: regrow_cases.py).

Each case starts a counter at a size it outgrows, through every path it names, and holds the result to:
  contents   the dump (8-byte counts) equals the numpy model key for key; records in (position, key) order under the final
             matrix; lookups of present and absent keys; histogram; the dump at counter length 1 and with -L / -U at the
             final in-slot counter width 2^cb
  statistics kmers == inserted == the model's total, distinct == the model's keys, regrows == final lsize - start lsize
  geometry   info() at the start and the end as the case claims; the reprobe limit of the start table carried
  restatement forced-size cases: header and body equal to oracle/_ref/jf_oracle count on the same files
  paths      every path of a case gives the same body"""
import os

import numpy as np
import pytest

import jfutil
import regrow_cases as R
import text_model

pytestmark = pytest.mark.gpu

TOP = (1 << 64) - 1


@pytest.fixture(scope="module")
def regrow_files(built, workdir):
    return R.write_files(workdir, sorted(R.FILES))


def _words(body, k, ocl):
    """Records of a body in file order -> ((n, nw) key words, counts)."""
    nw = 1 if k <= 32 else 2
    kb = (2 * k + 7) // 8
    r = np.frombuffer(body, np.uint8).reshape(-1, kb + ocl)
    kbuf = np.zeros((len(r), 8 * nw), np.uint8)
    kbuf[:, :kb] = r[:, :kb]
    cbuf = np.zeros((len(r), 8), np.uint8)
    cbuf[:, :ocl] = r[:, kb:]
    return kbuf.view("<u8").reshape(-1, nw), cbuf.view("<u8").reshape(-1)


def _clip_body(body, k, ocl_from, ocl_to):
    kb = (2 * k + 7) // 8
    keys, cnt = _words(body, k, ocl_from)
    r = np.frombuffer(body, np.uint8).reshape(-1, kb + ocl_from)
    c = np.minimum(cnt, np.uint64((1 << (8 * ocl_to)) - 1)).astype("<u8").view(np.uint8).reshape(-1, 8)[:, :ocl_to]
    return np.ascontiguousarray(np.concatenate((r[:, :kb], c), axis=1)).tobytes()


def _filter_body(body, k, ocl, lower, upper):
    kb = (2 * k + 7) // 8
    _, cnt = _words(body, k, ocl)
    r = np.frombuffer(body, np.uint8).reshape(-1, kb + ocl)
    return r[(cnt >= np.uint64(lower)) & (cnt <= np.uint64(upper))].tobytes()


def _ints(words):
    return text_model.as_ints(words)


def model_of(case, files):
    """-> (keys (n, nw) ascending, counts uint64, k-mers fed) of the table a case must end with (None for Bloom: see
    _check_bloom)."""
    k, can = case["k"], case["canonical"]
    if case["kind"] == "load":
        _, keys, cnt = R.load_body()
        order = np.argsort(keys)
        c2 = cnt[order].astype(object) * 2
        return keys[order].reshape(-1, 1), np.array([min(int(x), TOP) for x in c2], np.uint64), None
    sym = lambda names: text_model.stream([open(files[f], "rb").read() for f in names])
    if case["kind"] == "if":
        pk, _, _ = text_model.counts(sym(case["passes"][0]), k, can)
        uk, uc, total = text_model.counts(sym(case["passes"][1]), k, can)
        inv, _, _ = text_model._group(np.concatenate((pk, uk)))
        table = np.zeros(int(inv.max()) + 1, np.int64)
        table[inv[len(pk):]] = uc
        return pk, table[inv[:len(pk)]].astype(np.uint64), None
    keys, cnt, total = text_model.counts(sym(R.text_files(case)), k, can)
    return keys, cnt.astype(np.uint64), total


def _info_claim(info, claim, where):
    got = dict(slot_bits=info["slot_bits"], P=info["part_regions"], rec_bytes=info["part_rec_bytes"], lsize=info["lsize"])
    want = {x: claim[x] for x in claim if x != "window"}
    assert {x: got[x] for x in want} == want, where


def _feed(hc, case, path, files):
    """Feed every pass of a case (split further for passes_split); returns the info() after each pass of the case."""
    from jellyfish_b200 import HashCounter
    split = path.get("passes_split", 1)
    after = []
    for i, names in enumerate(case["passes"]):
        if case["kind"] == "if":
            hc.set_op(HashCounter.OP_PRIME if i == 0 else HashCounter.OP_UPDATE)
        if case["kind"] == "load":
            body = R.load_body()[0]
            rec = len(body) // len(R.load_body()[1])
            n = len(body) // rec
            if names[0] == "@load_reversed":
                body = np.frombuffer(body, np.uint8).reshape(n, rec)[::-1].tobytes()
            for j in range(split):
                hc.load_records(body[rec * (n * j // split):rec * (n * (j + 1) // split)], 8)
                hc.done()
        else:
            for j in range(split):
                for f in names:
                    data = open(files[f], "rb").read()
                    if split > 1:             # a share of the file's records
                        recs = data[1:].split(b"\n>")
                        data = b"".join(b">" + r + b"\n" for r in recs[len(recs) * j // split:len(recs) * (j + 1) // split])
                        data = data.replace(b"\n\n", b"\n")
                    hc.add_text(data)
                hc.done()
        after.append(hc.info())
    return after


def _run(case, pname, files, model):
    from jellyfish_b200 import HashCounter
    k, path = case["k"], dict(case["paths"][pname])
    kw = {x: v for x, v in path.items() if x != "passes_split"}
    if case["kind"] == "bloom":
        kw.update(bf_size=case["extra"]["bf_size"], bf_fp=case["extra"]["bf_fp"])
    where = (case["name"], pname)
    with HashCounter(1 << case["start_l"], 7, k=k, canonical=case["canonical"], reprobes=case["reprobes"], **kw) as hc:
        i0 = hc.info()
        g0 = R.part_geometry(k, case["start_l"], case["reprobes"], no_partition=kw.get("no_partition", False))
        claim0 = dict(case["start"]) if not kw.get("no_partition") else dict(slot_bits=case["start"]["slot_bits"], P=0, rec_bytes=0)
        _info_claim(i0, dict(claim0, lsize=case["start_l"]), where + ("start",))
        after = _feed(hc, case, path, files)
        st = hc.done()
        info = hc.info()
        L = info["lsize"]
        carried = g0["max_reprobe"]
        g = R.part_geometry(k, L, carried, no_partition=kw.get("no_partition", False))
        # geometry at the end: the case's claim where it makes one, the model of part_configure everywhere
        _info_claim(info, dict(slot_bits=g["slot_bits"], P=g["P"], rec_bytes=g["rec_bytes"]), where + ("end model",))
        if case["end"] is not None and not kw.get("no_partition"):
            _info_claim(info, case["end"], where + ("end",))
        if case["final_l"] is not None:
            assert L == case["final_l"], where
        for a, claim in zip(after, case["extra"].get("after_pass", [])):
            _info_claim(a, claim, where + ("after pass",))
        assert info["max_reprobe"] == g["max_reprobe"], where
        assert L > case["start_l"] and st["regrows"] == L - case["start_l"], (where, st["regrows"], L)
        if L == 2 * k:
            assert info["matrix_identity"] == 1, where
        body8 = hc.dump_records(out_counter_len=8)
        keys8, cnt8 = _words(body8, k, 8)
        # records in (original position, key) order under the final matrix
        pos = jfutil.positions(info, keys8, k).astype(np.uint64)
        d = np.diff(pos.astype(np.int64))
        assert np.all(d >= 0), where
        tie = np.flatnonzero(d == 0)
        if len(tie):
            assert np.all(text_model.less(keys8[tie], keys8[tie + 1])), where
        skeys, scnt = text_model.records_to_words(body8, k, 8)
        scnt = scnt.astype(np.uint64)                 # (counts of 2^63 and more)
        if model is not None:
            mkeys, mcnt, total = model
            assert len(skeys) == len(mkeys), (where, len(skeys), len(mkeys))
            assert np.array_equal(skeys, mkeys), where
            assert np.array_equal(scnt.astype(np.uint64), mcnt), where
            if case["kind"] == "count":
                assert st["kmers"] == st["inserted"] == total, (where, st)
                assert st["distinct"] == len(mkeys), (where, st)
        else:
            _check_bloom(case, files, skeys, scnt, where)
        _check_readers(hc, case, info, body8, skeys, scnt, where)
        hdr = hc.header()
        body4 = hc.dump_records()
    return dict(body8=body8, body4=body4, header=hdr, regrows=st["regrows"], lsize=L)


def _check_readers(hc, case, info, body8, skeys, scnt, where):
    from jellyfish_b200.engine import canonical_int
    k = case["k"]
    rng = np.random.default_rng(case["start_l"] * 977 + k)
    pick = rng.choice(len(skeys), size=min(3000, len(skeys)), replace=False)
    present = _ints(skeys[pick])
    assert hc.get_many(present) == [int(x) for x in scnt[pick]], where
    absent = []
    while len(absent) < 2000:
        x = int(rng.integers(0, 1 << 62)) | (int(rng.integers(0, 1 << 62)) << 62)
        x &= (1 << (2 * k)) - 1
        if case["canonical"]:
            x = canonical_int(x, k)
        absent.append(x)
    words = np.array([[(x >> (64 * w)) & TOP for w in range(skeys.shape[1])] for x in absent], np.uint64)
    _, ii, _ = np.intersect1d(np.ascontiguousarray(words).view([("", "<u8")] * skeys.shape[1]).ravel(),
                              np.ascontiguousarray(skeys).view([("", "<u8")] * skeys.shape[1]).ravel(), return_indices=True)
    got, hit = hc.get_many(absent), set(ii.tolist())
    assert all(got[i] == 0 for i in range(len(absent)) if i not in hit), where
    want = np.bincount(np.minimum(scnt, 63).astype(np.int64), minlength=64)
    assert hc.histogram(64) == want.tolist(), where
    assert hc.dump_records(out_counter_len=1) == _clip_body(body8, k, 8, 1), where
    cb = jfutil.geometry(k, info["lsize"], info["max_reprobe"])["cb"]
    lo = 1 << min(cb, 63)
    assert hc.dump_records(lower=lo, out_counter_len=8) == _filter_body(body8, k, 8, lo, TOP), where
    assert hc.dump_records(upper=lo - 1, out_counter_len=8) == _filter_body(body8, k, 8, 0, lo - 1), where


def _check_bloom(case, files, skeys, scnt, where):
    """count --bf-size: every count in {occ - 1, occ}, every key seen twice present, few singletons through."""
    occ_k, occ_c, _ = text_model.counts(text_model.stream([open(files[f], "rb").read() for f in R.text_files(case)]),
                                        case["k"], case["canonical"])
    inv, _, _ = text_model._group(np.concatenate((occ_k, skeys)))
    table = np.full(int(inv.max()) + 1, -1, np.int64)
    table[inv[:len(occ_k)]] = occ_c
    occ = table[inv[len(occ_k):]]
    assert np.all(occ >= 1), where                                    # only keys of the input
    assert np.all((scnt == occ) | (scnt == occ - 1)), where
    assert len(skeys) >= int((occ_c >= 2).sum()), where
    singles = int((occ_c == 1).sum())
    passed = len(skeys) - int((occ_c >= 2).sum())
    assert passed <= 3 * case["extra"]["bf_fp"] * singles + 50, (where, passed, singles)


def _oracle(case, files, workdir):
    out = os.path.join(workdir, "regrow_oracle_%s.jf" % case["name"])
    names = R.text_files(case)
    args = R.oracle_args(case)
    if case["kind"] == "if":
        args += ["--if", files[names[0]]]
        names = names[1:]
    if case["kind"] == "load":
        names = ["load_text"]
    jfutil.run([jfutil.ORACLE_C, "count"] + args + ["-o", out] + [files[f] for f in names], timeout=900)
    return jfutil.split_db(out)


@pytest.mark.parametrize("name", [c["name"] for c in R.CASES])
def test_doubling_case(name, regrow_files, workdir):
    case = R.BY_NAME[name]
    model = None if case["kind"] == "bloom" else model_of(case, regrow_files)
    runs = {p: _run(case, p, regrow_files, model) for p in case["paths"]}
    # across paths: the same body wherever the number of doublings agrees (always, for forced-size cases)
    first = next(iter(runs.values()))
    if case["kind"] != "bloom":
        for p, r in runs.items():
            if r["regrows"] == first["regrows"]:
                assert r["body8"] == first["body8"], (name, p)
    if case["final_l"] is None:
        return
    h, b = _oracle(case, regrow_files, workdir)
    for p, r in runs.items():
        if case["kind"] == "load":            # the matrix of the same draws: a text with as many keys, same start
            assert (r["header"]["size"], r["header"]["matrix1"]) == (h["size"], h["matrix1"]), (name, p)
            continue
        assert {x: r["header"][x] for x in jfutil.SEMANTIC_KEYS} == jfutil.semantic(h), (name, p)
        if case["kind"] != "bloom":
            assert r["body4"] == b, (name, p)
    if case["name"] == "into_direct_index":
        # the same text counted in a table created at 4^k slots
        from jellyfish_b200 import HashCounter
        with HashCounter(1 << 24, 7, k=case["k"], canonical=case["canonical"], **case["paths"]["k2_0"]) as hc:
            for f in R.text_files(case):
                hc.add_text(open(regrow_files[f], "rb").read())
                hc.done()
            assert hc.dump_records() == first["body4"]
            assert {x: hc.header()[x] for x in jfutil.SEMANTIC_KEYS} == {x: first["header"][x] for x in jfutil.SEMANTIC_KEYS}
