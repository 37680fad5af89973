"""Counting k-mers longer than 64 bases on the GPU (four-word keys, the wide slot form): every case of
tests/golden/golden_large_k.json byte for byte against the unmodified reference, the reference's own large_key.sh, `query -s`,
a Python-int model of a multi-Mbp count, the Python API, and inputs where every thread hits the same few keys."""
import collections
import json
import os
import random

import pytest

import gen
import jfutil

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = json.load(open(os.path.join(HERE, "golden", "golden_large_k.json")))


def _subst(args, inputs):
    return [inputs[a[1:-1]] if a.startswith("{") else a for a in args]


def _count(args, files, out):
    jfutil.run([jfutil.OUR_JF, "count"] + args + ["-o", out] + files)
    return jfutil.split_db(out)


@pytest.mark.parametrize("name", sorted(GOLDEN["cases"]))
def test_count_against_reference_golden(name, built, workdir, inputs):
    g = GOLDEN["cases"][name]
    db = os.path.join(workdir, "lk_%s.jf" % name)
    h, b = _count(_subst(g["args"], inputs), [inputs[i] for i in g["inputs"]], db)
    assert jfutil.semantic(h) == g["header"]
    assert jfutil.md5(b) == g["body_md5"]
    if "dump_c_md5" in g:
        assert jfutil.md5(jfutil.run([jfutil.OUR_JF, "dump", "-c", db]).stdout) == g["dump_c_md5"]
    if "histo" in g:
        assert jfutil.run([jfutil.OUR_JF, "histo", db]).stdout.decode() == g["histo"]
    if "query_md5" in g:         # query -s on the device: the database loaded back into a wide table
        q = jfutil.run([jfutil.OUR_JF, "query", "-s", inputs[g["query_file"]], db]).stdout
        assert jfutil.md5(q) == g["query_md5"]


@pytest.fixture(scope="module")
def seq1m(workdir):
    p = os.path.join(workdir, "seq1m_0_10001.fa")
    gen.generate_sequence_fasta(p + ".full", 1040104553, 1000000)
    with open(p + ".full", "rb") as f:
        lines = f.read().split(b"\n")
    with open(p, "wb") as f:
        f.write(b"\n".join(lines[:10001]) + b"\n")
    return p


@pytest.mark.parametrize("name", ["s2M", "s2k", "s2k_disk"])
def test_reference_large_key_sh(name, built, workdir, seq1m):
    g = GOLDEN["large_key"][name]
    db = os.path.join(workdir, "large_key_%s.jf" % name)
    h, b = _count(["-m", "100"] + g["args"], [seq1m], db)
    dump = jfutil.run([jfutil.OUR_JF, "dump", "-c", db]).stdout
    mers = b"".join(sorted(line.split(b" ")[0] + b"\n" for line in dump.splitlines()))
    assert jfutil.md5(mers) == g["sorted_mers_md5"] == "ded3925fe6bbaca10accc10d1bde11b5"
    assert jfutil.semantic(h) == g["header"]
    assert jfutil.md5(b) == g["body_md5"]


def _model(seq, k, canonical=True):
    """count of every canonical k-mer of a sequence without resets, with Python ints"""
    code = {65: 0, 67: 1, 71: 2, 84: 3}
    mask = (1 << (2 * k)) - 1
    f = r = 0
    out = collections.Counter()
    for i, ch in enumerate(seq):
        c = code[ch]
        f = ((f << 2) | c) & mask
        r = (r >> 2) | ((3 - c) << (2 * (k - 1)))
        if i >= k - 1:
            out[min(f, r) if canonical else f] += 1
    return out


def test_multi_mbp_count_against_python_model(built, workdir):
    from jellyfish_b200 import HashCounter
    seq = gen._seq(2000000, 77)
    seq = seq[:1500000] + seq[200000:700000]             # repeated stretch: counts of 2
    model = _model(seq, 100)
    with HashCounter(1 << 20, 7, k=100, canonical=True) as hc:
        hc.add_text(gen.fasta(seq))
        st = hc.done()
        assert st["kmers"] == len(seq) - 99
        assert st["distinct"] == len(model)
        path = os.path.join(workdir, "model100.jf")
        hc.dump(path)
        hist = hc.histogram(4)
        sample = random.Random(5).sample(sorted(model), 2000)
        assert hc.get_many(sample) == [model[x] for x in sample]
        assert hc.get_many([0, (1 << 200) - 1]) == [model.get(0, 0), model.get((1 << 200) - 1, 0)]
    h, b = jfutil.split_db(path)
    got = dict(jfutil.records(h, b))
    assert got == dict(model)
    hc_hist = collections.Counter(min(v, 3) for v in model.values())
    assert list(hist[1:4]) == [hc_hist[1], hc_hist[2], hc_hist[3]]


def test_python_api_round_trip(built, workdir):
    from jellyfish_b200 import HashCounter, load_database, int_to_mer, canonical_int, mer_to_int
    seq = gen._seq(50000, 78)
    model = _model(seq, 120)
    with HashCounter(1 << 16, 7, k=120, canonical=True) as hc:
        assert hc.key_words == 4
        hc.add_text(gen.fasta(seq))
        hc.done()
        path = os.path.join(workdir, "api120.jf")
        hc.dump(path)
        m = int_to_mer(next(iter(model)), 120)
        assert mer_to_int(m) == next(iter(model))
        rc = m[::-1].translate(str.maketrans("ACGT", "TGCA"))
        assert canonical_int(mer_to_int(rc), 120) == next(iter(model))
        assert hc.get_many([m, rc]) == [model[next(iter(model))]] * 2
    db = load_database(path)
    try:
        keys = sorted(model)[:500]
        assert db.get_many(keys) == [model[x] for x in keys]
        out = db.query_text(gen.fasta(seq[:5000])).decode().splitlines()
        assert len(out) == 5000 - 119
        assert all(int(c) == model[canonical_int(mer_to_int(x), 120)] for x, c in (line.split() for line in out))
    finally:
        db.close()


def test_hot_keys_period3_and_polya(built, workdir):
    """Every thread of the grid inserts the same three (period-3 repeat) or one (poly-A) k-mer: the claim / publish protocol
    of the wide form under contention, by ordinary use."""
    from jellyfish_b200 import HashCounter
    for unit, n in ((b"ACG", 3000000), (b"A", 2000000)):
        seq = (unit * (n // len(unit) + 1))[:n]
        with HashCounter(1 << 12, 7, k=100, canonical=True) as hc:
            hc.add_text(gen.fasta(seq))
            st = hc.done()
            path = os.path.join(workdir, "hot.jf")
            hc.dump(path)
        got = dict(jfutil.records(*jfutil.split_db(path)))
        model = _model(seq, 100)
        assert st["kmers"] == n - 99
        assert got == dict(model)


def test_iid_text_into_tiny_table_that_doubles(built, workdir, inputs):
    """High load and many doublings: the claim / publish protocol while the table fills, then regrow of wide slots."""
    db = os.path.join(workdir, "tiny100.jf")
    h, b = _count(["-m", "100", "-s", "1k", "-C", "-p", "10"], [inputs["plain1m.fa"]], db)
    assert h["size"] >= 1 << 20
    assert dict(jfutil.records(h, b)) == dict(_model(gen._seq(1000000, 2), 100))


def _fasta_model(data, k):
    """canonical k-mer counts of FASTA text: '>' at a line start opens a header line, any other non-base resets"""
    code = {65: 0, 67: 1, 71: 2, 84: 3, 97: 0, 99: 1, 103: 2, 116: 3}
    mask = (1 << (2 * k)) - 1
    out = collections.Counter()
    f = r = n = 0
    line_start, header = True, False
    for c in data:
        if c == 10:
            line_start = True
            continue
        if line_start:
            line_start = False
            header = c == 62
            if header:
                n = 0
        if header:
            continue
        if c in code:
            f = ((f << 2) | code[c]) & mask
            r = (r >> 2) | ((3 - code[c]) << (2 * (k - 1)))
            n += 1
            if n >= k:
                out[min(f, r)] += 1
        else:
            n = 0
    return out


def test_k100_across_the_reference_parser_buffer_boundary(built, workdir, inputs):
    """multi.fa at k = 100: the reference drops 138 k-mers that span one of its 4096-byte parser buffers (DESIGN.md 7a);
    every k-mer of the text is counted here."""
    db = os.path.join(workdir, "multi100.jf")
    h, b = _count(["-m", "100", "-s", "1M", "-C"], [inputs["multi.fa"]], db)
    assert dict(jfutil.records(h, b)) == dict(_fasta_model(open(inputs["multi.fa"], "rb").read(), 100))
