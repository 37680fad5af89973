"""The split of one file among ranks (jellyfish_b200/split.py) against the text model (tests/text_model.py), on the CPU.

FASTA: for every cut, the k-mers of the whole file in input order must be the concatenation, over the shares, of the k-mers
of [seam, end) without those of [seam, start) -- what a rank counts after jfgpu_seam.  FASTQ: wherever the newline check
passes, the k-mers of the shares concatenated must be those of the file, and a file built to fool the local rule must fail
the check.  The model's FASTA and FASTQ parsers are called directly, since a share need not start with '>' or '@'."""
import os
import random

import numpy as np
import pytest

import gen
import seam_corpus
import text_model as tm
from jellyfish_b200 import split

KS = (1, 2, 21, 31, 32, 33, 63, 64, 65, 100, 128)
SMALL = 6000              # files up to this size take every byte offset as a cut
MAX_BYTES = 400000        # (plain1m.fa adds nothing the 300 kb files do not cover, at several times their cost)


def _reader(data):
    return lambda off, n: data[off:off + n]


def _sym(data, fmt):
    d = np.frombuffer(data, np.uint8)
    body = (tm._fasta(d) if fmt == "fasta" else tm._fastq(d)) if len(d) else np.zeros(0, np.uint8)
    return np.concatenate(([tm.BREAK], body, [tm.BREAK])).astype(np.uint8)


def _kmers(data, fmt, k):
    return tm.kmers(_sym(data, fmt), k)


def _shares(data, fmt, starts, k):
    """Shares with the given starts (sorted, starts[0] = 0) and the planner's seams."""
    ends = list(starts[1:]) + [len(data)]
    rd = _reader(data)
    return [split.Share(fmt, split.fasta_seam_start(rd, s, k) if fmt == "fasta" and s < e else s, s, max(s, e))
            for s, e in zip(starts, ends)]


def _counted(data, share, k):
    """The k-mers rank counts: those of [seam, end) without those of [seam, start), which must be their prefix."""
    if share.start >= share.end:
        return None
    w = _kmers(data[share.seam:share.end], share.fmt, k)
    m = len(_kmers(data[share.seam:share.start], share.fmt, k)) if share.seam < share.start else 0
    return w[m:]


def _check(data, fmt, shares, k, full):
    parts = [p for p in (_counted(data, sh, k) for sh in shares) if p is not None]
    got = np.concatenate(parts) if parts else full[:0]
    assert got.shape == full.shape and np.array_equal(got, full), ([tuple(s) for s in shares], k)


def _fasta_inputs(tmp):
    files = gen.make_all(str(tmp))
    out = {n: open(p, "rb").read() for n, p in sorted(files.items()) if n.endswith(".fa")}
    out = {n: d for n, d in out.items() if 0 < len(d) <= MAX_BYTES}
    ev = seam_corpus.fasta_events(31, 0)
    rng = random.Random(17)
    for i in range(6):
        out["hostile%d" % i] = seam_corpus.hostile_fasta(4000 + 500 * i, rng, ev)
    out["dense"] = seam_corpus.dense_text({n: e for n, e in ev.items() if len(e) < 500}, 60000)[0]
    return out


@pytest.fixture(scope="module")
def fasta_inputs(tmp_path_factory):
    return _fasta_inputs(tmp_path_factory.mktemp("split_fa"))


@pytest.mark.parametrize("k", KS)
def test_fasta_every_cut(fasta_inputs, k):
    """Two shares cut at every byte offset (small files: every offset maps to a line start, each distinct one is checked;
    larger files: every line start in a seeded sample of offsets)."""
    rng = random.Random(k)
    for name, data in fasta_inputs.items():
        full = _kmers(data, "fasta", k)
        rd = _reader(data)
        offs = range(len(data) + 1) if len(data) <= SMALL else sorted(rng.sample(range(len(data)), 12))
        for s in sorted({split.share_start(rd, len(data), "fasta", a) for a in offs}):
            _check(data, "fasta", _shares(data, "fasta", [0, s], k), k, full)


@pytest.mark.parametrize("k", KS)
def test_fasta_worlds(fasta_inputs, k):
    for name, data in fasta_inputs.items():
        full = _kmers(data, "fasta", k)
        rd = _reader(data)
        for world in range(2, 9):
            shares = [split.plan_share(rd, len(data), "fasta", r, world, k) for r in range(world)]
            assert shares[0].start == 0 and shares[-1].end == len(data)
            for a, b in zip(shares, shares[1:]):
                assert a.end == b.start or (a.start >= a.end and b.start >= a.start)
            _check(data, "fasta", shares, k, full)


def test_fasta_tiny_files_leave_ranks_empty():
    data = b">x\nACGTACGTAC\n"
    shares = [split.plan_share(_reader(data), len(data), "fasta", r, 8, 5) for r in range(8)]
    assert sum(sh.end - sh.start for sh in shares) == len(data)
    assert sum(1 for sh in shares if sh.start < sh.end) <= 2


def _fastq_inputs(tmp):
    files = gen.make_all(str(tmp))
    names = ("reads.fq", "reads_dos.fq", "reads_noeol.fq", "reads_long.fq", "one_read.fq", "reads_q.fq", "reads_q_dos.fq")
    out = {n: open(files[n], "rb").read() for n in names}
    out["corpus"] = seam_corpus.fastq_text(200000, 31)
    out["corpus_dos"] = seam_corpus.fastq_text(100000, 33, eol=b"\r\n")
    return out


def _tallies(data, shares):
    return [(sh.end - sh.start, data[sh.start:sh.end].count(b"\n") if sh.start < sh.end else 0) for sh in shares]


@pytest.mark.parametrize("k", (1, 21, 31, 33, 64, 65, 128))
def test_fastq_shares(tmp_path_factory, k):
    inputs = _fastq_inputs(tmp_path_factory.mktemp("split_fq"))
    rng = random.Random(k)
    for name, data in inputs.items():
        full = _kmers(data, "fastq", k)
        rd = _reader(data)
        plans = [[split.plan_share(rd, len(data), "fastq", r, w, k) for r in range(w)] for w in range(2, 9)]
        for a in sorted(rng.sample(range(len(data)), min(len(data), 40))):
            plans.append(_shares(data, "fastq", [0, split.share_start(rd, len(data), "fastq", a)], k))
        for shares in plans:
            assert all(sh.seam == sh.start for sh in shares)
            if split.fastq_cuts_ok(_tallies(data, shares)):
                _check(data, "fastq", shares, k, full)


def test_fastq_check_catches_a_fooled_cut():
    """Sequence lines that start with '@', quality lines that start with '+' and header lines as long as the '+' lines: a cut
    that lands in a header finds the sequence line behind it, and the two records from there look whole."""
    rng = random.Random(3)
    recs = []
    for i in range(50):
        sq = b"@" + bytes(rng.choice(b"ACGT") for _ in range(40))
        recs.append(b"@r\n" + sq + b"\n+r\n+" + b"I" * (len(sq) - 1) + b"\n")
    data = b"".join(recs)
    rd = _reader(data)
    a = len(recs[0]) * 7 + 1                                  # inside the header of record 7
    s = split.share_start(rd, len(data), "fastq", a)
    assert s == len(recs[0]) * 7 + 3                          # the local rule takes the sequence line
    shares = _shares(data, "fastq", [0, s], 31)
    assert not split.fastq_cuts_ok(_tallies(data, shares))
    # cut in front of a header: the check passes and the count is exact
    s = split.share_start(rd, len(data), "fastq", len(recs[0]) * 7)
    shares = _shares(data, "fastq", [0, s], 31)
    assert split.fastq_cuts_ok(_tallies(data, shares))
    _check(data, "fastq", shares, 31, _kmers(data, "fastq", 31))


def test_empty_shares_are_not_checked():
    assert split.fastq_cuts_ok([(100, 12), (0, 0), (40, 3), (0, 0)])
    assert not split.fastq_cuts_ok([(100, 13), (40, 3)])


def test_plan_file_and_sniff(tmp_path):
    p = tmp_path / "a.fa"
    p.write_bytes(b">x\n" + b"ACGT" * 1000 + b"\n")
    assert split.plan_file(str(p), 0, 2, 21).start == 0
    sh = split.plan_file(str(p), 1, 2, 21)
    assert sh.fmt == "fasta" and sh.end == os.path.getsize(p)
    (tmp_path / "e.fa").write_bytes(b"")
    assert split.plan_file(str(tmp_path / "e.fa"), 1, 2, 21) is None
    (tmp_path / "z.gz").write_bytes(b"\x1f\x8b\x08\x00")
    with pytest.raises(ValueError):
        split.plan_file(str(tmp_path / "z.gz"), 0, 2, 21)


def test_pipes_are_not_split(tmp_path):
    """A FIFO or a process substitution can be read once, from its start: the commands give it whole to one rank."""
    p = tmp_path / "a.fa"
    p.write_bytes(b">x\nACGT\n")
    assert split.splittable(str(p))
    fifo = str(tmp_path / "fifo")
    os.mkfifo(fifo)
    assert not split.splittable(fifo)
    r, w = os.pipe()
    try:
        assert not split.splittable("/proc/self/fd/%d" % r)
    finally:
        os.close(r)
        os.close(w)
    assert not split.splittable(str(tmp_path / "missing.fa"))


def test_no_seam_in_front_of_a_header():
    data = b">a\n" + b"ACGT" * 30 + b"\n>b\n" + b"ACGT" * 30 + b"\n"
    s = data.index(b">b")
    assert split.fasta_seam_start(_reader(data), s, 31) == s
    assert split.fasta_seam_start(_reader(data), s + 4, 31) < s + 4
