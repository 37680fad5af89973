"""`count --sam` on the H100: SAM, gzip'd SAM and BAM files count as the FASTQ reads they hold.

The reference's SAM path hands each record's SEQ and qualities to the code of its FASTQ path
(mer_overlap_sequence_parser.hpp:220-253, whole_sequence_parser.hpp:192-208), so every FASTQ golden is also a SAM and a BAM
golden, byte for byte.  Corners the goldens do not reach are held to a model (sam_tools.sam_model_fastq) whose FASTQ the
engine counts on its FASTQ path, which the goldens pin to the reference.
"""
import gzip
import hashlib
import json
import os
import random
import subprocess

import pytest

import jfutil
import sam_tools
from cases import CASES, QUAL_CASES, BF_CASES

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = json.load(open(os.path.join(HERE, "golden", "golden.json")))
GOLDEN_QUAL = json.load(open(os.path.join(HERE, "golden", "golden_qual.json")))
GOLDEN_BF = json.load(open(os.path.join(HERE, "golden", "golden_bf.json")))

# the golden cases whose inputs are all 4-line FASTQ with "\n" line ends and a final newline
SAM_CASES = {n: CASES[n] for n in ("fq", "fq_k63", "fq_long")}
SAM_CASES.update({n: QUAL_CASES[n] for n in ("q_all_pass", "q_fq", "q_fq_hi", "q_long", "q_minq", "q_minq_dflt", "q_uniform")})
FORMS = ("sam", "sam.gz", "bam")


def _write_forms(workdir, inputs, name):
    """<name> as SAM, gzip'd SAM and BGZF-compressed BAM (cached in workdir)"""
    base = os.path.join(workdir, "samconv_" + name)
    if not os.path.exists(base + ".bam"):
        with open(inputs[name], "rb") as f:
            sam = sam_tools.fastq_to_sam(f.read())
        with open(base + ".sam", "wb") as f:
            f.write(sam)
        with open(base + ".sam.gz", "wb") as f:
            f.write(gzip.compress(sam))
        with open(base + ".bam", "wb") as f:
            f.write(sam_tools.bgzf(sam_tools.sam_to_bam(sam), block=50000))
    return {form: base + "." + form for form in FORMS}


def _count(workdir, tag, args, files=(), sams=()):
    db = os.path.join(workdir, "sam_%s.jf" % tag)
    cmd = [jfutil.OUR_JF, "count"] + list(args) + ["-o", db] + list(files)
    for s in sams:
        cmd += ["--sam", s]
    jfutil.run(cmd, timeout=900)
    return jfutil.split_db(db)


@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("name", sorted(SAM_CASES))
def test_sam_matches_fastq_golden(name, form, built, workdir, inputs):
    args, ins = SAM_CASES[name]
    g = GOLDEN.get(name) or GOLDEN_QUAL[name]
    sams = [_write_forms(workdir, inputs, i)[form] for i in ins]
    h, b = _count(workdir, "%s_%s" % (name, form.replace(".", "_")), args, sams=sams)
    assert jfutil.semantic(h) == g["header"]
    assert len(b) == g["body_len"] and jfutil.md5(b) == g["body_md5"]


@pytest.mark.parametrize("form", FORMS)
def test_sam_bloom_prefilter(form, built, workdir, inputs):
    """bf_fq: which first occurrences pass the filter depends on the insertion order, so (as for FASTQ) the header must be
    the golden one and every count in {occ - 1, occ}, where k-mers seen twice or more are present."""
    args, ins = BF_CASES["bf_fq"]
    sams = [_write_forms(workdir, inputs, i)[form] for i in ins]
    h, b = _count(workdir, "bf_fq_" + form.replace(".", "_"), args, sams=sams)
    assert jfutil.semantic(h) == GOLDEN_BF["bf_fq"]["header"]
    hr, br = _count(workdir, "bf_fq_occ", ["-m", "21", "-s", "1M", "-C"], files=[inputs[i] for i in ins])
    occ, got = dict(jfutil.records(hr, br)), dict(jfutil.records(h, b))
    assert set(got) <= set(occ)
    assert all(v in (occ[k], occ[k] - 1) for k, v in got.items())
    assert all(k in got for k, v in occ.items() if v > 1)


def test_sam_after_fasta_positionals(built, workdir, inputs):
    """FASTA positionals with --sam files: the same database as the SAM files' reads given as FASTQ."""
    args = ["-m", "21", "-s", "2M", "-C"]
    fa = [inputs["multi.fa"], inputs["plain.fa"]]
    sams = [_write_forms(workdir, inputs, "reads.fq")["bam"], _write_forms(workdir, inputs, "reads_q.fq")["sam"]]
    h1, b1 = _count(workdir, "mixed_sam", args, files=fa, sams=sams)
    h2, b2 = _count(workdir, "mixed_fq", args, files=fa + [inputs["reads.fq"], inputs["reads_q.fq"]])
    assert jfutil.semantic(h1) == jfutil.semantic(h2) and b1 == b2


@pytest.mark.parametrize("q", [None, "5"])
def test_sam_k100(q, built, workdir, inputs):
    """k = 100 (K1w, four-word keys): --sam against this engine's count of the same FASTQ (pinned by golden_large_k.json)."""
    args = ["-m", "100", "-s", "1M", "-C"] + (["-Q", q] if q else [])
    fq = inputs["reads_q.fq" if q else "reads.fq"]
    h1, b1 = _count(workdir, "k100_sam_%s" % q, args, sams=[_write_forms(workdir, inputs, os.path.basename(fq))["bam" if q else "sam"]])
    h2, b2 = _count(workdir, "k100_fq_%s" % q, args, files=[fq])
    assert jfutil.semantic(h1) == jfutil.semantic(h2) and b1 == b2 and b1


GEN_SEQ = os.path.join(jfutil.REF_DIR, "generate_sequence")


@pytest.mark.skipif(not os.path.exists(GEN_SEQ), reason="oracle/_ref/generate_sequence is not built")
@pytest.mark.parametrize("form", ["sam", "bam"])
def test_reference_sam_test_numbers(form, built, workdir):
    """The histo md5s the reference's tests/sam.sh publishes for seq10m.sam / .bam (count -m 20 -s 10M -C, and with -Q D)."""
    d = os.path.join(workdir, "seq10m")
    os.makedirs(d, exist_ok=True)
    fq = os.path.join(d, "seq10m.fq")
    if not os.path.exists(fq):
        jfutil.run([GEN_SEQ, "-q", "-o", os.path.join(d, "seq10m"), "-s", "1473540700", "10000000"], timeout=600)
    forms = {}
    for f in ("sam", "bam"):
        forms[f] = os.path.join(d, "seq10m." + f)
    if not os.path.exists(forms["bam"]):
        with open(fq, "rb") as f:
            sam = sam_tools.fastq_to_sam(f.read())
        with open(forms["sam"], "wb") as f:
            f.write(sam)
        with open(forms["bam"], "wb") as f:
            f.write(sam_tools.bgzf(sam_tools.sam_to_bam(sam)))
    for extra, want in (([], "8f8a71e04c27cd88918f11d44d9b3852"), (["-Q", "D"], "f0faf797cc55add8b6e88ab67bbcf19b")):
        db = os.path.join(d, "seq10m_%s%s.jf" % (form, "_qual" if extra else ""))
        jfutil.run([jfutil.OUR_JF, "count", "-m", "20", "-s", "10M", "-C"] + extra + ["-o", db, "--sam", forms[form]], timeout=900)
        histo = jfutil.run([jfutil.OUR_JF, "histo", db]).stdout
        assert hashlib.md5(histo).hexdigest() == want


def _corner_sam():
    rng = random.Random(7)

    def rec(seq, qual=None, tags=b"", name=b"r", eol=b"\n"):
        if qual is None:
            qual = bytes(rng.choice(b"!#+5?DIJ") for _ in seq) if seq != b"*" else b"*"
        return b"\t".join([name, b"0", b"chr1", b"1", b"60", b"*", b"*", b"0", b"0", seq, qual]) + tags + eol

    def bases(n, alphabet=b"ACGT"):
        return bytes(rng.choice(alphabet) for _ in range(n))
    return {
        "header_only": b"@HD\tVN:1.6\n@SQ\tSN:chr1\tLN:100\n",
        "empty": b"",
        "seq_star": rec(bases(80)) + rec(b"*") + rec(bases(60)),
        "qual_star": rec(bases(90), b"*") + rec(bases(70)) + rec(bases(3), b"*"),
        "iupac": rec(bases(120, b"ACGTacgtNRYKM=.U")) + rec(bases(150, b"ACGTacgt=.")) + rec(bases(40, b"acgt")),
        "long_tags": rec(bases(100), tags=b"\tXA:Z:" + b"x" * 3000 + b"\tNM:i:1") + rec(bases(50), tags=b"\t" + b"\t".join(b"T%d:i:1" % i for i in range(400))),
        "crlf": b"@HD\tVN:1.6\r\n" + rec(bases(100), eol=b"\r\n") + b"\r\n" + rec(bases(100), b"*", eol=b"\r\n") + rec(bases(60)),
        "no_final_newline": rec(bases(100)) + rec(bases(77))[:-1],
        "no_final_newline_qstar": rec(bases(100)) + rec(bases(77), b"*")[:-1],
        "late_headers_blank": rec(bases(100)) + b"@CO\tcomment\n\n" + rec(bases(100)) + b"\n\n@CO\tx\n" + rec(bases(30)),
        "tile_long_read": rec(bases(200)) + rec(bases(70000)) + rec(bases(40000, b"ACGTN")) + rec(bases(200)),
    }


CORNERS = _corner_sam()


@pytest.mark.parametrize("q", [None, "5"])
@pytest.mark.parametrize("name", sorted(CORNERS))
def test_sam_corners_against_model(name, q, built, workdir):
    sam = CORNERS[name]
    d = os.path.join(workdir, "corners")
    os.makedirs(d, exist_ok=True)
    sp, fp = os.path.join(d, name + ".sam"), os.path.join(d, name + ".fq")
    with open(sp, "wb") as f:
        f.write(sam)
    with open(fp, "wb") as f:
        f.write(sam_tools.sam_model_fastq(sam))
    args = ["-m", "17", "-s", "1M", "-C"] + (["-Q", q] if q else [])
    h1, b1 = _count(workdir, "corner_sam_%s_%s" % (name, q), args, sams=[sp])
    h2, b2 = _count(workdir, "corner_fq_%s_%s" % (name, q), args, files=[fp])
    assert jfutil.semantic(h1) == jfutil.semantic(h2)
    assert b1 == b2


def _seam_sam(inputs):
    with open(inputs["reads_q.fq"], "rb") as f:
        sam = sam_tools.fastq_to_sam(f.read())
    return sam


@pytest.mark.parametrize("form", ["sam", "bam"])
@pytest.mark.parametrize("q", [0, "5"])
def test_sam_feed_seams(form, q, built, inputs):
    """One file fed whole and cut at every offset of a window (inside the header and inside records), with staging
    buffers small enough that lines and records straddle batches and tiles: the same table."""
    from jellyfish_b200 import HashCounter
    sam = _seam_sam(inputs)
    data = sam if form == "sam" else sam_tools.sam_to_bam(sam)
    bam = form == "bam"

    def count(cuts, batch):
        with HashCounter(1 << 20, 7, k=21, canonical=True, max_batch_bytes=batch, min_qual=q) as hc:
            pos = 0
            for i, c in enumerate(list(cuts) + [len(data)]):
                hc.add_sam_text(data[pos:c], begin=i == 0, end=c == len(data), bam=bam)
                pos = c
            hc.done()
            return hc.dump_records()
    whole = count([], 0)
    assert whole
    assert count([], 4096) == whole
    # a window over the header and the first records, then one around a record boundary further in
    for c in list(range(1, 700, 23)) + list(range(len(data) // 2 - 300, len(data) // 2 + 300, 29)):
        assert count([c], 8192) == whole, "cut at %d" % c
    assert count(range(1000, len(data), 977), 2048) == whole


@pytest.mark.parametrize("bam", [False, True])
def test_sam_format_flag_on_first_feed_only(bam, built, inputs):
    """The format given with FILE_BEGIN holds for the later feeds of the file, which may leave the flag out (as the CLI does)."""
    from jellyfish_b200 import HashCounter, _lib as L
    sam = _seam_sam(inputs)
    data = sam_tools.sam_to_bam(sam) if bam else sam
    flag = L.FORMAT_BAM if bam else L.FORMAT_SAM
    with HashCounter(1 << 20, 7, k=21, canonical=True) as hc:
        hc.add_sam_text(data, bam=bam)
        hc.done()
        whole = hc.dump_records()
    with HashCounter(1 << 20, 7, k=21, canonical=True) as hc:
        cuts = list(range(0, len(data), 100003)) + [len(data)]
        for i in range(len(cuts) - 1):
            piece = data[cuts[i]:cuts[i + 1]]
            fl = (L.FILE_BEGIN | flag if i == 0 else 0) | (L.FILE_END if i == len(cuts) - 2 else 0)
            hc._check(hc._lib.jfgpu_feed(hc._h, piece, len(piece), fl))
        hc.done()
        assert hc.dump_records() == whole


def test_sam_device_feed_seams(built, inputs):
    """SAM text in device memory: the same table whole, cut anywhere across feeds, and in small batches."""
    import torch
    from jellyfish_b200 import HashCounter
    sam = _seam_sam(inputs)
    dev = torch.frombuffer(bytearray(sam), dtype=torch.uint8).cuda()

    def count(cuts, batch):
        with HashCounter(1 << 20, 7, k=21, canonical=True, max_batch_bytes=batch) as hc:
            pos = 0
            for i, c in enumerate(list(cuts) + [len(sam)]):
                # (each piece copied to an aligned buffer of its own: jfgpu_feed_device takes 16-byte aligned text)
                piece = dev[pos:c].clone()
                hc.add_device_text(piece.data_ptr(), c - pos, begin=i == 0, end=c == len(sam), sam=True)
                torch.cuda.synchronize()
                pos = c
            hc.done()
            return hc.dump_records()
    whole = count([], 0)
    with HashCounter(1 << 20, 7, k=21, canonical=True) as hc:
        hc.add_sam_text(sam)
        hc.done()
        assert hc.dump_records() == whole
    assert count([], 4096) == whole
    for c in list(range(1, 400, 13)) + [len(sam) // 2 + i for i in range(0, 400, 17)]:
        assert count([c], 8192) == whole, "cut at %d" % c


def _bad_inputs():
    good = b"r\t0\tchr1\t1\t60\t4M\t*\t0\t0\tACGT\tIIII\n"
    bam = sam_tools.sam_to_bam(good * 3)
    return {
        "few_fields": (good + b"r\t0\tchr1\t1\t60\t4M\t*\t0\tACGT\tIIII\n" + good, "fewer than 11 fields"),
        "qual_len": (good + b"r\t0\tchr1\t1\t60\t4M\t*\t0\t0\tACGT\tIII\n", "SEQ and QUAL of different lengths"),
        "bam_truncated": (sam_tools.bgzf(bam[:-5]), "Truncated BAM record"),
    }


@pytest.mark.parametrize("name", sorted(_bad_inputs()))
def test_sam_malformed_input_fails(name, built, workdir):
    data, msg = _bad_inputs()[name]
    p = os.path.join(workdir, "bad_" + name)
    with open(p, "wb") as f:
        f.write(data)
    out = os.path.join(workdir, "bad_%s.jf" % name)
    r = subprocess.run([jfutil.OUR_JF, "count", "-m", "5", "-s", "1k", "-o", out, "--sam", p], stderr=subprocess.PIPE)
    assert r.returncode != 0
    assert msg in r.stderr.decode()
    assert not os.path.exists(out)


def test_sam_flags_refused_where_they_do_not_apply(built):
    """Both format flags at once, and BAM from device memory, are argument errors."""
    from jellyfish_b200 import HashCounter, JellyfishError, _lib as L
    with HashCounter(1 << 16, 7, k=21) as hc:
        with pytest.raises(JellyfishError) as ei:
            hc._check(hc._lib.jfgpu_feed(hc._h, b"", 0, L.FILE_BEGIN | L.FORMAT_SAM | L.FORMAT_BAM))
        assert ei.value.code == L.ERR_ARG
        with pytest.raises(JellyfishError) as ei:
            hc._check(hc._lib.jfgpu_feed_device(hc._h, None, 0, L.FILE_BEGIN | L.FORMAT_BAM, None))
        assert ei.value.code == L.ERR_ARG
