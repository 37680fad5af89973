"""tests/kmer_model.py, the exact counter the full-size bench steps are checked against (test_gpu_bench_exact.py), held to
the C restatement of the reference (oracle/_ref/jf_oracle) on the CPU.

The texts have the synthetic layout of the bench ('>read1', 70-column lines).  Chunks of a few kilobases put hundreds of
seams into every text, and eight partitions split every digest.  The table sizes put many keys on the same original
position, so the (position, key) order of a dump is checked within positions too; one of them doubles."""
import os

import pytest
import torch

import gen
import jfutil
import kmer_model as km

P = 8
CHUNK = 3000

# (k, bases, -s): k = 21 in a table that doubles twice, k = 31 and 63 at loads near 0.5
CASES = [(21, 120_000, "32k"), (31, 100_000, "256k"), (63, 60_000, "128k")]


@pytest.fixture(scope="module")
def oracle_dbs(built, tmp_path_factory):
    """k -> (FASTA bytes, oracle header, oracle body)."""
    d = tmp_path_factory.mktemp("kmer_model")
    out = {}
    for k, n, size in CASES:
        text = gen.fasta(gen._seq(n, 9000 + k))
        fa = os.path.join(str(d), "m%d.fa" % k)
        with open(fa, "wb") as f:
            f.write(text)
        db = os.path.join(str(d), "m%d.jf" % k)
        jfutil.run([jfutil.ORACLE_C, "count", "-m", str(k), "-s", size, "-C", "-o", db, fa])
        h, b = jfutil.split_db(db)
        out[k] = (text, h, b)
    return out


def _digest(k, header, body, cuts):
    """StreamDigest of a body fed in slices cut at the given byte offsets."""
    m = header["matrix1"]
    assert not m["identity"]
    sd = km.StreamDigest(k, header["size"], m["columns"], header["counter_len"], P, "cpu")
    edges = [0] + list(cuts) + [len(body)]
    for a, b in zip(edges[:-1], edges[1:]):
        sd.feed(torch.frombuffer(bytearray(body[a:b]), dtype=torch.uint8) if b > a else torch.zeros(0, dtype=torch.uint8))
    return sd.finish()


def test_mix_is_splitmix64_finalizer():
    def ref(x):
        x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9 & (2 ** 64 - 1)
        x = (x ^ (x >> 27)) * 0x94D049BB133111EB & (2 ** 64 - 1)
        return x ^ (x >> 31)
    xs = [0, 1, 2 ** 63, 2 ** 64 - 1, 0x9E3779B97F4A7C15, 0x0123456789ABCDEF, 2 ** 42 - 1]
    got = km.mix(torch.tensor([km._s64(x) for x in xs], dtype=torch.int64)).tolist()
    assert [g & (2 ** 64 - 1) for g in got] == [ref(x) for x in xs]


def test_keys_are_the_engines_canonical_integers():
    """Random k-mers and the all-A / all-T extremes, against engine.canonical_int (Python ints)."""
    from jellyfish_b200.engine import canonical_int, mer_to_int
    for k in (1, 21, 31, 32, 33, 63, 64):
        mers = [b"A" * k, b"T" * k] + [gen._seq(k, 77 * k + i) for i in range(40)]
        w = km.mers_words(torch.tensor([list(m) for m in mers], dtype=torch.uint8), k).tolist()
        got = [sum((x & (2 ** 64 - 1)) << (64 * j) for j, x in enumerate(row)) for row in w]
        assert got == [canonical_int(mer_to_int(m.decode()), k) for m in mers], k


@pytest.mark.parametrize("k", [c[0] for c in CASES])
def test_model_digests_equal_the_oracle_body(oracle_dbs, k):
    text, h, body = oracle_dbs[k]
    assert h["size"] > 1 << 15 or k != 21          # the k = 21 table has doubled
    recs = jfutil.records(h, body)
    # queries: keys of the body, keys that are absent
    present = [x for x, _ in recs[::97]]
    absent = km.random_words(300, k, 5, "cpu")
    wq = torch.cat([torch.tensor(jfutil.key_words(present, k).astype("int64")), absent])
    model = km.count(torch.frombuffer(bytearray(text), dtype=torch.uint8), k, P=P, chunk_bases=CHUNK, queries=wq)
    n_bases = len(text) - len(b">read1\n") - text.count(b"\n") + 1
    assert model.n_kmers == n_bases - k + 1
    sd = _digest(k, h, body, [])
    assert sd.n_disorder == 0 and sd.n_records == len(recs) == model.distinct()
    assert km.differing_partitions(model, sd) == []
    assert (model.digest[:, 0] > 0).all()             # every partition holds keys
    assert model.digest[:, 1].sum() == model.n_kmers
    d = dict(recs)
    expect = [d[x] for x in present]
    expect += [d.get(sum((v & (2 ** 64 - 1)) << (64 * j) for j, v in enumerate(row)), 0) for row in absent.tolist()]
    assert model.query_counts.tolist() == expect
    assert sum(1 for c in expect[len(present):] if c == 0) > 250
    # partitions gathered three at a time (several passes over the text) give the same model
    again = km.count(torch.frombuffer(bytearray(text), dtype=torch.uint8), k, P=P, chunk_bases=CHUNK, queries=wq, per_pass=3)
    assert torch.equal(again.digest, model.digest) and torch.equal(again.hist, model.hist)
    assert torch.equal(again.query_counts, model.query_counts)


@pytest.mark.parametrize("k", [c[0] for c in CASES])
def test_stream_digest_accepts_the_oracle_order_in_any_slices(oracle_dbs, k):
    text, h, body = oracle_dbs[k]
    rec = (2 * k + 7) // 8 + h["counter_len"]
    whole = _digest(k, h, body, [])
    cuts = sorted({1, rec, rec + 3, len(body) // 3, len(body) // 3 + 5, len(body) - 1})
    sliced = _digest(k, h, body, cuts)
    assert sliced.n_disorder == 0 and sliced.n_records == whole.n_records
    assert torch.equal(sliced.digest, whole.digest) and torch.equal(sliced.hist, whole.hist)
    # positions: as jfutil.positions computes them from the header's matrix
    keys = [x for x, _ in jfutil.records(h, body)[:500]]
    a = torch.frombuffer(bytearray(body[:500 * rec]), dtype=torch.uint8).view(500, rec)
    pos = whole.positions(a)
    info = {"size": h["size"], "matrix_identity": False, "matrix_columns": h["matrix1"]["columns"], "matrix_c": h["matrix1"]["c"]}
    assert pos.tolist() == jfutil.positions(info, keys, k).astype("int64").tolist()
    assert len(set(pos.tolist())) < len(keys)          # keys share original positions: the key breaks ties


def _records(h, k, body):
    rec = (2 * k + 7) // 8 + h["counter_len"]
    return [body[i:i + rec] for i in range(0, len(body), rec)]


@pytest.mark.parametrize("k", [c[0] for c in CASES])
def test_stream_digest_rejects_a_tampered_body(oracle_dbs, k):
    text, h, body = oracle_dbs[k]
    model = km.count(torch.frombuffer(bytearray(text), dtype=torch.uint8), k, P=P, chunk_bases=CHUNK)
    recs = _records(h, k, body)
    kb = (2 * k + 7) // 8
    i = len(recs) // 2
    # two neighbours swapped: the same digests, out of order
    sw = list(recs)
    sw[i], sw[i + 1] = sw[i + 1], sw[i]
    sd = _digest(k, h, b"".join(sw), [len(body) // 2])
    assert sd.n_disorder >= 1 and km.differing_partitions(model, sd) == []
    # one count changed: in order, one partition differs
    ch = list(recs)
    ch[i] = ch[i][:kb] + (int.from_bytes(ch[i][kb:], "little") + 1).to_bytes(h["counter_len"], "little")
    sd = _digest(k, h, b"".join(ch), [])
    assert sd.n_disorder == 0 and len(km.differing_partitions(model, sd)) == 1
    # one record stored twice: equal (position, key), and its partition differs
    du = recs[:i + 1] + recs[i:]
    sd = _digest(k, h, b"".join(du), [(i + 1) * len(recs[0])])
    assert sd.n_disorder == 1 and sd.first_disorder[0] == i + 1 and len(km.differing_partitions(model, sd)) == 1


def test_model_without_overlap_between_chunks_is_caught(oracle_dbs, monkeypatch):
    """The model's seams matter: chunks that do not share k - 1 bases lose k-mers, and the digests say so."""
    k = 21
    text, h, body = oracle_dbs[k]
    orig = km._chunks

    def no_overlap(t, k_, chunk_bases):
        for codes in orig(t, k_, chunk_bases):
            yield codes[k_ - 1:] if codes.numel() > 2 * (k_ - 1) else codes
    monkeypatch.setattr(km, "_chunks", no_overlap)
    model = km.count(torch.frombuffer(bytearray(text), dtype=torch.uint8), k, P=P, chunk_bases=CHUNK)
    assert km.differing_partitions(model, _digest(k, h, body, []))
