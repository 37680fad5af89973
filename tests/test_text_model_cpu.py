"""Pin tests/text_model.py, the numpy model of the text contract, to the C restatement oracle/_ref/jf_oracle (and, where it
was built, to the reference itself).  No GPU.

The model's symbol stream does not depend on k: the k-mers it gives for k > 64 (which neither program counts) are
windows of the same stream that these tests pin at every k up to 64, so k = 65..128 is pinned with it."""
import os
import random

import numpy as np
import pytest

import gen
import jfutil
import seam_corpus as sc
import text_model as tm

KS = (1, 5, 17, 31, 32, 33, 63, 64)


def _oracle(tmp, files, k, canonical, extra=(), exe=None):
    out = os.path.join(tmp, "o.jf")
    n_bytes = sum(os.path.getsize(f) for f in files)
    size = max(1024, 2 * n_bytes)
    cmd = [exe or jfutil.ORACLE_C, "count", "-m", str(k), "-s", str(size), "-o", out] + (["-C"] if canonical else []) + list(extra)
    if exe is None:
        cmd += ["--out-counter-len", "8"]
    jfutil.run(cmd + list(files))
    h, b = jfutil.split_db(out)
    return tm.records_to_words(b, k, h["counter_len"])


def _check(tmp, datas, k, canonical, min_qual=0, label="", exe=None):
    files = []
    for i, d in enumerate(datas):
        p = os.path.join(tmp, "in%d" % i)
        with open(p, "wb") as f:
            f.write(d)
        files.append(p)
    extra = ["-Q", chr(min_qual)] if min_qual else []
    keys, cnt = _oracle(tmp, files, k, canonical, extra, exe)
    mk, mc, _ = tm.counts(tm.stream(datas, min_qual), k, canonical)
    assert len(mk) == len(keys) and np.array_equal(mk, keys) and np.array_equal(mc, cnt), \
        "%s k=%d%s: model %d distinct / %d k-mers, oracle %d / %d" % (label, k, " -C" if canonical else "", len(mk), mc.sum(), len(keys), cnt.sum())


@pytest.fixture(scope="module")
def oracle_built(built):
    if not os.path.exists(jfutil.ORACLE_C):
        pytest.skip("oracle not built")


GEN_FILES = ["plain.fa", "dos.fa", "noeol.fa", "lower.fa", "multi.fa", "multi2.fa", "empty.fa", "header_only.fa",
             "dangling.fa", "one_per_line.fa", "blank_runs.fa", "long_header.fa", "cr_mid.fa", "oneline.fa", "polya.fa",
             "repeat.fa", "reads.fq", "reads_dos.fq", "reads_noeol.fq", "reads_long.fq", "one_read.fq", "reads_ml.fq",
             "reads_q.fq", "reads_q_dos.fq"]


@pytest.mark.parametrize("name", GEN_FILES)
def test_model_matches_oracle_on_gen_inputs(name, oracle_built, inputs, tmp_path):
    data = open(inputs[name], "rb").read()
    for i, k in enumerate(KS):
        # (the oracle simulates the table slot by slot: files of 100 KB and more take one orientation per k)
        for canonical in (False, True) if len(data) < 100000 else (i % 2 == 1,):
            _check(str(tmp_path), [data], k, canonical, label=name)


def test_model_matches_oracle_across_files(oracle_built, inputs, tmp_path):
    datas = [open(inputs[n], "rb").read() for n in ("cr_mid.fa", "empty.fa", "header_only.fa", "noeol.fa", "reads_noeol.fq", "multi2.fa")]
    for k in (5, 31, 64):
        _check(str(tmp_path), datas, k, True, label="files")


@pytest.mark.parametrize("name,q", [("reads_q.fq", "5"), ("reads_q_dos.fq", "5"), ("reads.fq", "@"), ("reads_ml.fq", "7"),
                                    ("dos.fa", "I"), ("multi.fa", "I"), ("cr_mid.fa", "I")])
def test_model_matches_oracle_min_quality(name, q, oracle_built, inputs, tmp_path):
    data = open(inputs[name], "rb").read()
    for k in (5, 17, 31, 33, 64):
        _check(str(tmp_path), [data], k, k % 2 == 1, min_qual=ord(q), label=name)


def _hostile(i):
    """Seeded hostile text number i: FASTA from the seam vocabulary, 4-line FASTQ (DOS or not), or FASTQ for -Q."""
    rng = random.Random(1000 + i)
    form = ("fasta", "fastq", "fastq_q", "fasta_q")[i % 4]
    k = rng.choice(KS)
    events = sc.fasta_events(k, rng.choice((0, 300)))
    n = rng.randrange(500, 6000)
    if form.startswith("fasta"):
        return form, k, sc.hostile_fasta(n, rng, events)
    low = b"!#%\x80\xf0" if form == "fastq_q" else b""
    return form, k, sc.fastq_text(n, k, seed=i, eol=rng.choice((b"\n", b"\r\n")), low=low, long_every=0)


@pytest.mark.parametrize("block", range(8))
def test_model_matches_oracle_on_hostile_texts(block, oracle_built, tmp_path):
    for i in range(block * 25, block * 25 + 25):
        form, k, data = _hostile(i)
        mq = ord("5") if form.endswith("_q") else 0
        _check(str(tmp_path), [data], k, i % 3 == 0, min_qual=mq, label="hostile %d (%s)" % (i, form))


def test_model_matches_reference(oracle_built, tmp_path):
    """A dozen hostile texts through the reference's own `count`, away from its 4096-byte buffer artefacts (DESIGN.md
    section 7a): texts shorter than one buffer, one thread."""
    if not os.path.exists(jfutil.REF_JF):
        pytest.skip("reference not built")
    for i in range(12):
        rng = random.Random(50 + i)
        k = (5, 17, 31)[i % 3]
        events = sc.fasta_events(k, 0)
        data = sc.hostile_fasta(rng.randrange(300, 3500), rng, events) if i % 2 == 0 else \
            sc.fastq_text(rng.randrange(300, 3500), k, seed=i, eol=rng.choice((b"\n", b"\r\n")))
        _check(str(tmp_path), [data[:4000]], k, True, label="reference %d" % i, exe=jfutil.REF_JF)


def test_model_symbols_edge_cases():
    """The stream itself on texts small enough to read."""
    B = tm.BREAK
    s = lambda t, q=0: tm.symbols(t, q).tolist()
    assert s(b"") == [B]
    assert s(b">only") == [B, B, B]
    assert s(b">h\nAC\r\r\nG\n") == [B, B, 0, 1, 2, B]                  # line-end '\r' run dropped, lines joined
    assert s(b">h\nA\rC\n") == [B, B, 0, B, 1, B]                        # mid-line '\r' resets
    assert s(b">h\nA\n\r\r\n\n\rC\n") == [B, B, 0, 1, B]                  # blank lines and leading '\r' skipped
    assert s(b">h\nA\n\r>x\nC") == [B, B, 0, B, 1, B]                     # '>' after leading '\r' opens a header
    assert s(b">h\nA\xc1\xe7C") == [B, B, 0, B, B, 1, B]                  # high bytes are not bases
    assert s(b"@r\nAC\r\n+\r\n!!\r\n@s\nG\n+\n!\n") == [B, 0, 1, B, 2, B]
    assert s(b">h\nA\rC\n", ord("!")) == [B, B, 0, B, 1, B]
    assert s(b">h\nAC\r\nG\n", ord("!")) == [B, B, 0, 1, B, 2, B]        # -Q: a line-end '\r' is a byte of the line
    assert s(b"@r\nACGT\n+\n!5!5\n", ord("5")) == [B, B, B, 1, B, 3, B]
