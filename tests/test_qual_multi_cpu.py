"""`count_multi` under -Q and --if without a device: the command line's checks and messages (those of the single-GPU
`count`), FASTA shares that start on header lines (jellyfish_b200.split, headers=True) against a brute-force model, and the
pieces of a FASTQ share cut behind whole records (ShareReader, records=True) on random FASTQ."""
import ctypes as C
import random

import pytest

from jellyfish_b200 import split


def _parse(argv, capsys):
    from jellyfish_b200.count_multi import parse_args
    with pytest.raises(SystemExit) as ex:
        parse_args(argv)
    return ex.value.code, capsys.readouterr().err


def test_parse_args_takes_the_quality_switches_and_if():
    from jellyfish_b200.count_multi import parse_args
    a = parse_args(["-m", "21", "-s", "1M", "-Q", "5", "--if", "a.fa", "--if", "b.fq", "x.fq"])
    assert a.min_qual == ord("5") and a.if_files == ["a.fa", "b.fq"] and a.files == ["x.fq"]
    a = parse_args(["-m", "17", "-s", "1M", "--min-quality", "20", "--quality-start", "33", "x.fq"])
    assert a.min_qual == 53
    a = parse_args(["-m", "15", "-s", "1M", "--min-quality", "6", "x.fq"])
    assert a.min_qual == 64 + 6
    a = parse_args(["-m", "21", "-s", "1M", "--min-qual-char", "!", "--sam", "x.sam"])
    assert a.min_qual == ord("!") and a.sam == ["x.sam"]
    a = parse_args(["-m", "21", "-s", "1M", "x.fa"])
    assert a.min_qual == 0 and a.if_files == []
    # --min-quality is applied after -Q (jf_cli.cc)
    assert parse_args(["-m", "21", "-s", "1M", "-Q", "5", "--min-quality", "1", "--quality-start", "33", "x"]).min_qual == 34
    a = parse_args(["-m", "40", "-s", "1M", "-Q", "3", "--bf-size", "1M", "x.fq"])
    assert a.min_qual == ord("3") and a.bf_size == 1000000


@pytest.mark.parametrize("argv,msg", [
    (["-Q", "ab"], "Error: [-Q, --min-qual-char] must be one character.\n"),
    (["-Q", ""], "Error: [-Q, --min-qual-char] must be one character.\n"),
    (["-Q", " "], "Error: Quality character ' ' is outside of the range [!, ~]\n"),
    (["-Q", "\x7f"], "Error: Quality character '\x7f' is outside of the range [!, ~]\n"),
    (["--min-quality", "1", "--quality-start", "32"], "Error: Quality start 32 is outside the range [33, 126]\n"),
    (["--min-quality", "1", "--quality-start", "127"], "Error: Quality start 127 is outside the range [33, 126]\n"),
    (["--min-quality", "63"], "Error: Min quality 63 is outside the range [0, 62]\n"),
    (["--min-quality", "-1", "--quality-start", "33"], "Error: Min quality -1 is outside the range [0, 93]\n"),
    (["-Q", "5", "--bf-size", "1M", "--bc", "x.bc"], "Error: Switches [--bf-size] and [--bc] conflict\n"),
])
def test_parse_args_refuses_with_the_single_gpu_messages(argv, msg, capsys):
    code, err = _parse(["-m", "21", "-s", "1M"] + argv + ["x.fq"], capsys)
    assert code == 1 and err == msg


def _random_fasta(rng, n_records, eol=b"\n"):
    out = []
    for _ in range(n_records):
        out.append(b">" + bytes(rng.choice(b"ab>\r ") for _ in range(rng.randrange(0, 6))) + eol)
        for _ in range(rng.randrange(0, 5)):
            out.append(bytes(rng.choice(b"ACGTN>\r") for _ in range(rng.randrange(0, 30))) + eol)
    return b"".join(out)


def _header_model(data, a):
    if a <= 0:
        return 0
    for q in range(a, len(data)):
        if data[q - 1:q] == b"\n" and data[q:q + 1] == b">":
            return q
    return len(data)


@pytest.mark.parametrize("seed", range(6))
def test_fasta_header_cuts_match_a_brute_force_model(seed, monkeypatch):
    rng = random.Random(seed)
    data = _random_fasta(rng, rng.randrange(1, 40), eol=rng.choice([b"\n", b"\r\n"]))
    if seed % 2:
        monkeypatch.setattr(split, "WINDOW", 7)          # (windows far shorter than a line: every window seam is crossed)
    rd = lambda off, n: data[off:off + n]
    for a in range(0, len(data) + 2):
        assert split.share_start(rd, len(data), "fasta", a, headers=True) == _header_model(data, a), a
    for world in (1, 2, 3, 4, 8, 64):
        shares = [split.plan_share(rd, len(data), "fasta", r, world, 21, headers=True) for r in range(world)]
        assert shares[0].start == 0 and shares[-1].end == len(data)
        for s, t in zip(shares, shares[1:]):
            assert s.end == t.start or (s.start == s.end and t.start >= s.start)
        for s in shares:
            assert s.seam == s.start                      # no seam: a share starts on a header (or is empty)
            assert s.start == s.end or s.start == 0 or data[s.start - 1:s.start + 1] == b"\n>"


class _HostMemory(object):
    """Pageable stand-ins for the pinned buffers of ShareReader (no device here)."""

    def __init__(self):
        self.bufs = {}

    def jfgpu_host_alloc(self, n):
        b = C.create_string_buffer(n)
        self.bufs[C.addressof(b)] = b
        return C.addressof(b)

    def jfgpu_host_free(self, p):
        self.bufs.pop(p, None)


def _random_fastq(rng, n_reads, eol=b"\n", longest=300):
    out = []
    for i in range(n_reads):
        ln = rng.randrange(0, longest)
        out.append(b"@r%d" % i + eol + bytes(rng.choice(b"ACGTN") for _ in range(ln)) + eol + b"+" + eol +
                   bytes(rng.choice(b"!#5@IJ+") for _ in range(ln)) + eol)
    return b"".join(out)


def _read_pieces(path, share, piece_bytes, records):
    from jellyfish_b200 import distributed
    reader = distributed.ShareReader(path, share, piece_bytes, records=records)
    reader._lib = _HostMemory()
    pieces = []
    try:
        for i in range(reader.n_pieces):
            hptr, n, begin, end = reader.read(i)
            reader.prefetch(i + 1)
            pieces.append(C.string_at(hptr, n))
            reader.release(i)
    finally:
        reader.close()
    return pieces


@pytest.mark.parametrize("seed", range(4))
def test_fastq_pieces_end_behind_whole_records(seed, tmp_path):
    pytest.importorskip("numpy")
    import jellyfish_b200._lib as L
    import os
    if not os.path.exists(L.LIB_PATH):
        pytest.skip("libjfgpu.so is not built")
    rng = random.Random(seed)
    data = _random_fastq(rng, 400, eol=b"\r\n" if seed % 2 else b"\n")
    path = str(tmp_path / "r.fq")
    with open(path, "wb") as f:
        f.write(data)
    ends = set()
    lines = 0
    for p, c in enumerate(data):
        if c == 10:
            lines += 1
            if lines % 4 == 0:
                ends.add(p + 1)
    for world in (1, 2, 3):
        for piece_bytes in (6000, 9001, 1 << 20):
            for r in range(world):
                share = split.plan_file(path, r, world, 21)
                pieces = _read_pieces(path, share, piece_bytes, True)
                assert b"".join(pieces) == data[share.start:share.end]
                # the share starts on a record; every piece but the last ends behind one and none is longer than piece_bytes
                assert share.start == 0 or share.start in ends
                at = share.start
                for i, p in enumerate(pieces):
                    at += len(p)
                    assert len(p) <= piece_bytes
                    if i < len(pieces) - 1:
                        assert at in ends, (world, piece_bytes, r, i)
                    assert p.count(b"\n") % 4 == 0 or i == len(pieces) - 1


def test_fastq_record_longer_than_the_slack_is_refused(tmp_path):
    import jellyfish_b200._lib as L
    import os
    if not os.path.exists(L.LIB_PATH):
        pytest.skip("libjfgpu.so is not built")
    data = b"@a\n" + b"A" * 50000 + b"\n+\n" + b"I" * 50000 + b"\n" + b"@b\nAC\n+\nII\n"
    path = str(tmp_path / "long.fq")
    with open(path, "wb") as f:
        f.write(data)
    share = split.plan_file(path, 0, 1, 21)
    with pytest.raises(ValueError, match="no FASTQ record ends"):
        _read_pieces(path, share, 40000, True)
