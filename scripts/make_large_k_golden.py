#!/usr/bin/env python
"""Regenerate the goldens of k-mers longer than 64 bases from the UNMODIFIED reference (oracle/_ref/jellyfish and
oracle/_ref/ref_matrix, built by `make -C oracle all` where the reference sources are present):

  tests/golden/golden_large_k.json
    "cases":     `count` at k = 65..128 over the inputs of tests/gen.py (semantic header keys, body md5; for some also the
                 md5 of `dump -c`, `histo` and `query -s`)
    "large_key": the reference's own tests/large_key.sh: the first 10001 lines of seq1m_0.fa counted with -m 100 -s 2M,
                 -s 2k and -s 2k --disk; `dump -c | cut -d' ' -f1 | sort` has the md5 that script publishes
    "matrices":  hash matrices of 130..256 columns drawn by the reference library
    "host":      outputs of the reference's dump / query / info / histo / stats / merge on the two small k = 100
                 databases tests/golden/large_k_a.bin and large_k_b.bin (written here, by the reference's count)

    python scripts/make_large_k_golden.py
"""
import json
import os
import shutil
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import gen  # noqa: E402
import jfutil  # noqa: E402

LARGE_KEY_MD5 = "ded3925fe6bbaca10accc10d1bde11b5"      # tests/large_key.sh of the reference

# name -> (count switches, inputs, extra outputs: d = dump -c, h = histo, q = query -s of the listed file).  multi.fa is
# counted at k = 65, 96 and 128 only: at k = 100 the reference loses 138 k-mers that span one of its 4096-byte parser
# buffer boundaries (DESIGN.md section 7a; tests/test_gpu_large_k.py checks that case against a model instead)
CASES = {
    "k65": (["-m", "65", "-s", "1M"], ["plain.fa"], "dh"),
    "k65C_multi_files": (["-m", "65", "-s", "1M", "-C"], ["multi.fa", "multi2.fa"], "dhq"),
    "k96C_dos": (["-m", "96", "-s", "1M", "-C"], ["dos.fa"], "h"),
    "k96_noeol_lower": (["-m", "96", "-s", "1M"], ["noeol.fa", "lower.fa"], ""),
    "k100_one_per_line": (["-m", "100", "-s", "1M"], ["one_per_line.fa", "blank_runs.fa"], "d"),
    "k100C_fastq": (["-m", "100", "-s", "1M", "-C"], ["reads.fq", "reads_dos.fq"], "dhq"),
    "k100C_long_header": (["-m", "100", "-s", "256k", "-C"], ["long_header.fa", "cr_mid.fa", "oneline.fa"], ""),
    "k128C": (["-m", "128", "-s", "1M", "-C"], ["plain.fa", "multi.fa"], "dhq"),
    "k128_multi": (["-m", "128", "-s", "1M"], ["multi.fa"], ""),
    "k100C_grow": (["-m", "100", "-s", "2k", "-C"], ["plain.fa"], "h"),               # several doublings
    "k80_grow_p20": (["-m", "80", "-s", "1k", "-p", "20"], ["multi.fa"], ""),
    "k100C_disk": (["-m", "100", "-s", "64k", "-C", "--disk"], ["plain.fa", "reads.fq"], "d"),   # spills, then merges
    "k100C_ocl1": (["-m", "100", "-s", "1M", "-C", "--out-counter-len", "1"], ["polya.fa", "repeat.fa"], "d"),
    "k100C_LU": (["-m", "100", "-s", "1M", "-C", "-L", "2", "-U", "40"], ["repeat.fa", "plain.fa", "dos.fa"], ""),
    "k100C_text": (["-m", "100", "-s", "1M", "-C", "--text"], ["reads.fq", "one_per_line.fa"], ""),
    "k100C_if": (["-m", "100", "-s", "1M", "-C", "--if", "{noeol.fa}"], ["dos.fa", "reads.fq", "plain.fa"], "h"),
    "k100C_Q": (["-m", "100", "-s", "1M", "-C", "-Q", "5"], ["reads_q.fq", "reads_q_dos.fq"], "h"),
    "k72_Q_quality": (["-m", "72", "-s", "1M", "--min-quality", "20", "--quality-start", "33"], ["reads_q.fq"], ""),
}
MATRICES = [(10, 130, 0), (17, 160, 0), (22, 200, 1), (30, 256, 0), (31, 256, 0), (40, 192, 0), (62, 256, 2), (64, 250, 0)]


def ref(*args, **kw):
    return jfutil.run([jfutil.REF_JF] + list(args), **kw).stdout


def subst(args, inputs):
    return [inputs[a[1:-1]] if a.startswith("{") else a for a in args]


def large_key_input(path):
    """The first 10001 lines of the reference's seq1m_0.fa (generate_sequence -v -o seq1m -s 1040104553 1000000)."""
    with tempfile.TemporaryDirectory() as d:
        gen.generate_sequence_fasta(os.path.join(d, "seq1m_0.fa"), 1040104553, 1000000)
        with open(os.path.join(d, "seq1m_0.fa"), "rb") as f:
            lines = f.read().split(b"\n")
    with open(path, "wb") as f:
        f.write(b"\n".join(lines[:10001]) + b"\n")


def scrub_header(path, tag):
    """Replace where and when a database was written (host name, directory, time, command line) by fixed values, keeping
    the header's length: the fixture then says nothing about the machine that made it."""
    with open(path, "rb") as f:
        data = f.read()
    hlen = int(data[:9])
    h = json.loads(data[9:9 + hlen].rstrip(b"\0").decode())
    h.update({"hostname": "host", "pwd": "/data", "time": "2026-01-01T00:00:00", "exe_path": "jellyfish",
              "cmdline": ["count", "-m", "100", "-t", "1", "-s", "4k", "-C", "-o", "large_k_%s.jf" % tag, "small_%s.fa" % tag]})
    raw = json.dumps(h, separators=(",", ":"), sort_keys=True).encode()
    assert len(raw) <= hlen
    with open(path, "wb") as f:
        f.write(data[:9] + raw + b"\0" * (hlen - len(raw)) + data[9 + hlen:])


def sorted_mers_md5(dump_c):
    return jfutil.md5(b"".join(sorted(line.split(b" ")[0] + b"\n" for line in dump_c.splitlines())))


def main():
    out = {"cases": {}, "large_key": {}, "matrices": [], "host": {}}
    with tempfile.TemporaryDirectory() as d:
        inputs = gen.make_all(d)
        for name, (args, ins, extra) in CASES.items():
            db = os.path.join(d, name + ".jf")
            ref("count", "-t", "1", *subst(args, inputs), "-o", db, *[inputs[i] for i in ins])
            h, b = jfutil.split_db(db)
            c = {"args": args, "inputs": ins, "header": jfutil.semantic(h), "body_md5": jfutil.md5(b)}
            if "d" in extra:
                c["dump_c_md5"] = jfutil.md5(ref("dump", "-c", db))
            if "h" in extra:
                c["histo"] = ref("histo", db).decode()
            if "q" in extra:
                c["query_file"] = "reads.fq"
                c["query_md5"] = jfutil.md5(ref("query", "-s", inputs["reads.fq"], db))
            out["cases"][name] = c
            print(name, c["body_md5"])
        seq = os.path.join(d, "seq1m_0.fa")
        large_key_input(seq)
        for name, args in (("s2M", ["-s", "2M"]), ("s2k", ["-s", "2k"]), ("s2k_disk", ["-s", "2k", "--disk"])):
            db = os.path.join(d, "lk_%s.jf" % name)
            ref("count", "-m", "100", "-t", "1", *args, "-o", db, seq)
            md5 = sorted_mers_md5(ref("dump", "-c", db))
            assert md5 == LARGE_KEY_MD5, (name, md5)
            h, b = jfutil.split_db(db)
            out["large_key"][name] = {"args": args, "sorted_mers_md5": md5, "header": jfutil.semantic(h), "body_md5": jfutil.md5(b)}
        # two small k = 100 databases with the same size and matrix (both the first draw), for the CPU readers
        small = {}
        for tag, seed in (("a", 501), ("b", 502)):
            fa = os.path.join(d, "small_%s.fa" % tag)
            with open(fa, "wb") as f:
                f.write(gen.fasta(gen._seq(700, seed) + gen._seq(300, 600), line=60) + gen.fasta(gen._seq(200, 600) * 3, name=b"rep"))
            db = os.path.join(ROOT, "tests", "golden", "large_k_%s.bin" % tag)
            ref("count", "-m", "100", "-t", "1", "-s", "4k", "-C", "-o", db, fa)
            scrub_header(db, tag)
            small[tag] = db
            shutil.copy(fa, os.path.join(d, "q_%s.fa" % tag))
            out["host"]["fasta_" + tag] = open(fa).read()
        a, b = small["a"], small["b"]
        mers = []
        for line in ref("dump", "-c", a).decode().splitlines()[:5]:
            m = line.split()[0]
            rc = m[::-1].translate(str.maketrans("ACGT", "TGCA"))
            mers += [m, rc]
        mers += ["A" * 100, "ACGT" * 25, "ACGT" * 24, "ACGTN" * 20]
        hs = out["host"]
        hs["query_mers"] = mers
        for tag, db in small.items():
            hs[tag] = {
                "dump_md5": jfutil.md5(ref("dump", db)),
                "dump_ct_md5": jfutil.md5(ref("dump", "-c", "-t", db)),
                "dump_L2_md5": jfutil.md5(ref("dump", "-c", "-L", "2", db)),
                "query": ref("query", db, *mers).decode(),
                "query_s_md5": jfutil.md5(ref("query", "-s", os.path.join(d, "q_%s.fa" % tag), db)),
                "info": ref("info", db).decode(),
                "info_cmd": ref("info", "-c", db).decode(),
                "histo": ref("histo", db).decode(),
                "stats": ref("stats", db).decode(),
            }
        for op, flags in (("sum", []), ("min", ["--min"]), ("max", ["--max"])):
            m = os.path.join(d, "merged_%s.jf" % op)
            ref("merge", *flags, "-o", m, a, b)
            hm, bm = jfutil.split_db(m)
            hs["merge_" + op] = {"header": jfutil.semantic(hm), "body_md5": jfutil.md5(bm)}
        m = os.path.join(d, "merged_j.txt")
        ref("merge", "--jaccard", "-o", m, a, b)
        hs["merge_jaccard"] = open(m).read()
    for r, c, skip in MATRICES:
        cols = [int(x) for x in subprocess.check_output([os.path.join(jfutil.REF_DIR, "ref_matrix"), str(r), str(c), str(skip)]).split()]
        assert len(cols) == c
        out["matrices"].append({"r": r, "c": c, "skip": skip, "columns": cols})
    path = os.path.join(ROOT, "tests", "golden", "golden_large_k.json")
    with open(path, "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")
    print("wrote %s: %d cases" % (path, len(out["cases"])))


if __name__ == "__main__":
    main()
