"""`query -s` on the GPU and databases loaded back into a table (jfgpu_load_records, jfgpu_query).

The golden cases come from the reference's own `query -s` (tests/golden/golden_query.json, scripts/make_query_golden.py):
every database is first rebuilt with `jellyfish-b200 count` and checked against the reference's, so that a mismatch
blames the stage that made it."""
import collections
import json
import os
import subprocess

import numpy as np
import pytest

import gen
import jfutil

pytestmark = pytest.mark.gpu

GOLDEN = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "golden_query.json")))


@pytest.fixture(scope="module")
def dbs(built, workdir, inputs):
    """name -> path of every golden database, written by jellyfish-b200 count."""
    out = {}
    for name, g in GOLDEN["dbs"].items():
        p = os.path.join(workdir, "q_%s.jf" % name)
        jfutil.run([jfutil.OUR_JF, "count"] + g["args"] + ["-o", p] + [inputs[i] for i in g["inputs"]])
        out[name] = p
    return out


def _query_cli(db, files):
    return jfutil.run([jfutil.OUR_JF, "query"] + sum([["-s", f] for f in files], []) + [db]).stdout


@pytest.mark.parametrize("i", range(len(GOLDEN["queries"])),
                         ids=["%s-%s" % (q["db"], "+".join(q["files"])) for q in GOLDEN["queries"]])
def test_query_cli_against_reference_golden(i, dbs, inputs):
    q = GOLDEN["queries"][i]
    g = GOLDEN["dbs"][q["db"]]
    h, b = jfutil.split_db(dbs[q["db"]])
    assert jfutil.semantic(h) == g["header"] and jfutil.md5(b) == g["body_md5"], "the database differs from the reference's"
    out = _query_cli(dbs[q["db"]], [inputs[f] for f in q["files"]])
    assert out.count(b"\n") == q["lines"]
    assert jfutil.md5(out) == q["md5"]


def _kmer_ints(codes, k):
    """forward and reverse-complement 2-bit packed k-mers (first base most significant) of a code array (k <= 32)."""
    n = len(codes) - k + 1
    fw = np.zeros(n, dtype=np.uint64)
    rc = np.zeros(n, dtype=np.uint64)
    for i in range(k):
        c = codes[i:i + n].astype(np.uint64)
        fw |= c << np.uint64(2 * (k - 1 - i))
        rc |= (np.uint64(3) - c) << np.uint64(2 * i)
    return fw, rc


def test_query_20mbp_against_numpy(built, workdir):
    """No reference involved: a 20 Mbp single-record FASTA queried against a database of an overlapping text."""
    k = 21
    seq = gen._seq(26000000, 5)
    q_fa, d_fa, db = (os.path.join(workdir, n) for n in ("q20m.fa", "d20m.fa", "d20m.jf"))
    with open(q_fa, "wb") as f:
        f.write(gen.fasta(seq[:20000000]))
    with open(d_fa, "wb") as f:
        f.write(gen.fasta(seq[12000000:26000000]) + gen.fasta(seq[15000000:16000000], name=b"again"))
    jfutil.run([jfutil.OUR_JF, "count", "-m", str(k), "-s", "32M", "-C", "-o", db, d_fa])
    h, b = jfutil.split_db(db)
    recs = jfutil.records(h, b)
    keys = np.array([r[0] for r in recs], dtype=np.uint64)
    vals = np.array([r[1] for r in recs], dtype=np.uint64)
    order = np.argsort(keys)
    keys, vals = keys[order], vals[order]
    codes = np.frombuffer(b"\x00" * 256, dtype=np.uint8).copy()
    codes[list(b"ACGT")] = [0, 1, 2, 3]
    c = codes[np.frombuffer(seq[:20000000], dtype=np.uint8)]
    fw, rc = _kmer_ints(c, k)
    can = np.minimum(fw, rc)
    at = np.minimum(np.searchsorted(keys, can), len(keys) - 1)
    want = np.where(keys[at] == can, vals[at], 0)

    out = np.frombuffer(_query_cli(db, [q_fa]), dtype=np.uint8)
    ends = np.flatnonzero(out == ord("\n"))
    assert len(ends) == len(can)
    starts = np.concatenate(([0], ends[:-1] + 1))
    mers = out[starts[:, None] + np.arange(k)]
    shift = np.uint64(2) * (np.uint64(k - 1) - np.arange(k, dtype=np.uint64))
    got_codes = ((can[:, None] >> shift) & np.uint64(3)).astype(np.uint8)
    assert np.array_equal(mers, np.frombuffer(b"ACGT", dtype=np.uint8)[got_codes])
    assert np.all(out[starts + k] == ord(" "))
    ndig = ends - starts - k - 1
    assert ndig.min() >= 1
    got = np.zeros(len(can), dtype=np.uint64)
    for d in range(int(ndig.max())):
        has = ndig > d
        got[has] = got[has] * np.uint64(10) + (out[starts[has] + k + 1 + d] - ord("0")).astype(np.uint64)
    assert np.array_equal(got, want)
    assert (want > 0).sum() > len(want) // 3 and (want == 0).sum() > len(want) // 3       # both present and absent k-mers


def test_batch_seams_give_identical_bytes(dbs, inputs):
    from jellyfish_b200 import load_database
    texts = [open(inputs[f], "rb").read() for f in ("dos.fa", "reads.fq", "reads_dos.fq", "multi.fa", "one_per_line.fa")]
    outs = []
    for mbb in (4096, 65536 + 13, 0):
        with load_database(dbs["k31"], max_batch_bytes=mbb) as hc:
            outs.append([hc.query_text(t) for t in texts])
            # the same text in two calls, cut inside a line and inside a FASTQ record
            outs[-1].append(b"".join(hc.query_text(t[:len(t) // 2 + 7], begin=True, end=False) +
                                     hc.query_text(t[len(t) // 2 + 7:], begin=False, end=True) for t in texts))
    assert outs[0] == outs[1] == outs[2]
    assert outs[2][-1] == b"".join(outs[2][:-1])
    cli = [_query_cli(dbs["k31"], [inputs[f]]) for f in ("dos.fa", "reads.fq", "reads_dos.fq", "multi.fa", "one_per_line.fa")]
    assert cli == outs[2][:-1]


def _file_records(path):
    h, b = jfutil.split_db(path)
    return h, collections.Counter(jfutil.records(h, b))


@pytest.mark.parametrize("name", sorted(GOLDEN["dbs"]))
def test_loaded_database_dumps_its_records_and_histogram(name, dbs):
    from jellyfish_b200 import load_database
    h, want = _file_records(dbs[name])
    with load_database(dbs[name]) as hc:
        body = hc.dump_records(out_counter_len=h["counter_len"])
        assert collections.Counter(jfutil.records(h, body)) == want
        hist = hc.histogram(10002)
    got = {c: n for c, n in enumerate(hist) if n}
    ref = {int(a): int(n) for a, n in (l.split() for l in GOLDEN["dbs"][name]["histo"].splitlines())}
    assert got == ref


def test_load_that_regrows_keeps_every_count(dbs):
    from jellyfish_b200 import load_database
    h, want = _file_records(dbs["k31"])
    with load_database(dbs["k31"], size=1024) as hc:
        assert hc.done()["regrows"] >= 8
        assert collections.Counter(jfutil.records(h, hc.dump_records(out_counter_len=h["counter_len"]))) == want


def test_header_size_does_not_size_the_table(dbs, workdir):
    from jellyfish_b200 import load_database
    from jellyfish_b200.engine import write_header
    h2, body = jfutil.split_db(dbs["k17C"])
    big = os.path.join(workdir, "big_header.jf")
    with open(big, "wb") as f:
        write_header(f, dict(h2, size=1 << 31))
        f.write(body)
    with load_database(big) as hc:
        assert hc.size() < (1 << 24)
        assert collections.Counter(jfutil.records(h2, hc.dump_records(out_counter_len=h2["counter_len"]))) == \
            collections.Counter(jfutil.records(h2, body))


def test_query_leaves_the_table_as_it_was(dbs, inputs):
    from jellyfish_b200 import load_database
    with load_database(dbs["k17C"]) as hc:
        before = jfutil.md5(hc.dump_records())
        st = hc.done()
        n = hc.query_text(open(inputs["reads.fq"], "rb").read(), sink="discard")
        assert n == GOLDEN["queries"][[q["files"] for q in GOLDEN["queries"]].index(["reads.fq"])]["lines"]
        assert jfutil.md5(hc.dump_records()) == before
        st2 = hc.done()
        assert {k: st2[k] for k in ("kmers", "inserted", "distinct")} == {k: st[k] for k in ("kmers", "inserted", "distinct")}


def test_load_records_rejects_partial_records_and_bad_counter_lengths(dbs):
    from jellyfish_b200 import HashCounter, JellyfishError
    from jellyfish_b200 import _lib as L
    h, b = jfutil.split_db(dbs["k17C"])
    with HashCounter(1 << 20, k=17, canonical=True) as hc:
        for body, cl in ((b[:-1], h["counter_len"]), (b, 0), (b, 9)):
            with pytest.raises(JellyfishError) as ei:
                hc.load_records(body, cl)
            assert ei.value.code == L.ERR_ARG and str(ei.value)


def test_query_cli_errors(built, workdir, inputs, dbs):
    bad = os.path.join(workdir, "bad_first_byte.fa")
    with open(bad, "wb") as f:
        f.write(b"xACGT\n")
    r = subprocess.run([jfutil.OUR_JF, "query", "-s", bad, dbs["k17C"]], stdout=subprocess.PIPE, stderr=subprocess.PIPE)
    assert r.returncode != 0 and r.stderr.strip()
    bc = os.path.join(workdir, "q.bc")
    jfutil.run([jfutil.OUR_JF, "bc", "-m", "17", "-s", "1M", "-C", "-o", bc, inputs["multi.fa"]])
    txt = os.path.join(workdir, "q_text.jf")
    jfutil.run([jfutil.OUR_JF, "count", "-m", "17", "-s", "1M", "-C", "--text", "-o", txt, inputs["multi.fa"]])
    for db in (bc, txt):
        r = subprocess.run([jfutil.OUR_JF, "query", "-s", inputs["plain.fa"], db], stdout=subprocess.PIPE, stderr=subprocess.PIPE)
        assert r.returncode != 0 and b"Unsupported format" in r.stderr and not r.stdout


def test_query_files_matches_the_cli(dbs, inputs):
    from jellyfish_b200 import load_database
    files = [inputs[f] for f in ("plain.fa", "reads.fq", "multi2.fa", "empty.fa", "dos.fa")]
    got = []
    with load_database(dbs["k40C"]) as hc:
        n = hc.query_files(files, got.append, chunk=100000)
    out = b"".join(got)
    assert n == out.count(b"\n")
    assert out == _query_cli(dbs["k40C"], files)
