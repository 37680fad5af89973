"""The host side of `count --sam` (no device): the test's own SAM / BAM / BGZF writers, and the CLI's reader of --sam files
(`jellyfish-b200 inputs --sam`, the bytes `count` hands to the engine) checked against Python's gzip, with its errors."""
import gzip
import os
import struct
import subprocess

import pytest

import jfutil
import sam_tools

FQ = b"".join(b"@r%d\n%s\n+\n%s\n" % (i, b"ACGTTGCA"[i % 8:] * 20, b"I" * (160 - i % 8 * 20)) for i in range(300))


def _inputs(args, **kw):
    return subprocess.run([jfutil.OUR_JF, "inputs", "--marks"] + args, stdout=subprocess.PIPE, stderr=subprocess.PIPE, **kw)


def _bam_records(bam):
    """(seq, qual) of every record of an uncompressed BAM stream (SAM specification 4.2)."""
    assert bam[:4] == b"BAM\1"
    l_text = struct.unpack_from("<i", bam, 4)[0]
    p = 8 + l_text
    n_ref = struct.unpack_from("<i", bam, p)[0]
    p += 4
    for _ in range(n_ref):
        p += 4 + struct.unpack_from("<i", bam, p)[0] + 4
    out = []
    while p < len(bam):
        bs, = struct.unpack_from("<I", bam, p)
        l_name, = struct.unpack_from("<B", bam, p + 12)
        n_cig, = struct.unpack_from("<H", bam, p + 16)
        l_seq, = struct.unpack_from("<i", bam, p + 20)
        s = p + 36 + l_name + 4 * n_cig
        seq = "".join("=ACMGRSVTWYHKDBN"[(bam[s + i // 2] >> (0 if i & 1 else 4)) & 15] for i in range(l_seq))
        q = bam[s + (l_seq + 1) // 2: s + (l_seq + 1) // 2 + l_seq]
        out.append((seq.encode(), bytes((c + 33) & 255 for c in q)))
        p += 4 + bs
    assert p == len(bam)
    return out


def test_writers_round_trip():
    sam = sam_tools.fastq_to_sam(FQ)
    recs = [ln.split(b"\t") for ln in sam.split(b"\n") if ln and not ln.startswith(b"@")]
    assert {int(r[1]) for r in recs} == {0, 4, 16, 256}
    assert all(len(r) > 11 for r in recs)
    reads = sam_tools.parse_fastq(FQ)
    assert [(r[9], r[10]) for r in recs] == [(s, q) for _, s, q in reads]
    assert _bam_records(sam_tools.sam_to_bam(sam)) == [(s, q) for _, s, q in reads]
    z = sam_tools.bgzf(sam_tools.sam_to_bam(sam), block=1000)
    assert gzip.decompress(z) == sam_tools.sam_to_bam(sam)
    assert z.endswith(sam_tools.BGZF_EOF)


def test_model_rules():
    m = sam_tools.sam_model_fastq(b"@HD\n\nr\t0\t*\t0\t0\t*\t*\t0\t0\tAcgU=\t*\r\nr\t0\t*\t0\t0\t*\t*\t0\t0\t*\t*\n"
                                  b"r\t0\t*\t0\t0\t*\t*\t0\t0\tAC\t!!\tXX:Z:a")
    assert m == b"@\nAcgNN\n+\n     \n@\nAC\n+\n!!\n"
    with pytest.raises(ValueError):
        sam_tools.sam_model_fastq(b"r\t0\t*\t0\t0\t*\t*\t0\tAC\t!!\n")
    with pytest.raises(ValueError):
        sam_tools.sam_model_fastq(b"r\t0\t*\t0\t0\t*\t*\t0\t0\tAC\t!\n")


@pytest.mark.parametrize("chunk", [64 << 20, 4096, 777])
def test_reader_inflates_like_python(chunk, built, tmp_path):
    sam = sam_tools.fastq_to_sam(FQ * 20)
    bam = sam_tools.sam_to_bam(sam)
    files = {"a.sam": (sam, sam), "a.sam.gz": (gzip.compress(sam) + gzip.compress(sam[:100]), sam + sam[:100]),
             "a.bam": (sam_tools.bgzf(bam, block=3001), bam), "b.bam": (sam_tools.bgzf(bam), bam)}
    paths = []
    for name, (data, _) in files.items():
        (tmp_path / name).write_bytes(data)
        paths.append(str(tmp_path / name))
        if data[:2] == b"\x1f\x8b":
            assert gzip.decompress(data) == files[name][1]
    r = _inputs(["--chunk", str(chunk)] + sum((["--sam", p] for p in paths), []))
    assert r.returncode == 0, r.stderr
    assert r.stdout == b"".join(want for _, want in files.values())
    begins = [ln for ln in r.stderr.decode().splitlines() if " begin" in ln]
    assert [("bam" in ln, "sam" in ln.split()[-1]) for ln in begins] == [(False, True), (False, True), (True, False), (True, False)]


def test_sam_files_come_after_the_others(built, tmp_path):
    (tmp_path / "x.fa").write_bytes(b">a\nACGT\n")
    (tmp_path / "y.sam").write_bytes(b"r\t0\t*\t0\t0\t*\t*\t0\t0\tAC\t!!\n")
    r = _inputs(["--sam", str(tmp_path / "y.sam"), str(tmp_path / "x.fa")])
    assert r.returncode == 0 and r.stdout == b">a\nACGT\nr\t0\t*\t0\t0\t*\t*\t0\t0\tAC\t!!\n"


def test_reader_errors(built, tmp_path):
    cram = tmp_path / "x.cram"
    cram.write_bytes(b"CRAM\x03\x00" + b"\0" * 100)
    r = _inputs(["--sam", str(cram)])
    assert r.returncode != 0 and b"CRAM input is not supported" in r.stderr
    r = _inputs(["--sam", str(tmp_path / "missing.sam")])
    assert r.returncode != 0 and b"Can't open SAM file '" in r.stderr
    z = sam_tools.bgzf(sam_tools.sam_to_bam(sam_tools.fastq_to_sam(FQ)), block=2000)
    (tmp_path / "t.bam").write_bytes(z[:len(z) // 2])
    r = _inputs(["--sam", str(tmp_path / "t.bam")])
    assert r.returncode != 0 and b"Truncated BGZF block" in r.stderr
    g = gzip.compress(sam_tools.fastq_to_sam(FQ))
    (tmp_path / "t.sam.gz").write_bytes(g[:len(g) // 2])
    r = _inputs(["--sam", str(tmp_path / "t.sam.gz")])
    assert r.returncode != 0 and b"Truncated gzip stream" in r.stderr
    bad = bytearray(z)
    bad[40] ^= 0xff                                       # inside the first block's deflate data
    (tmp_path / "c.bam").write_bytes(bytes(bad))
    r = _inputs(["--sam", str(tmp_path / "c.bam")])
    assert r.returncode != 0 and b"Corrupt BGZF block" in r.stderr
