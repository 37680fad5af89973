#!/usr/bin/env python
"""Differential fuzz of the readers of jellyfish-b200 (dump, histo, stats, query, merge: plain CPU code in
jellyfish_b200/csrc/host/jf_cli.cc, except `query -s`, which runs on the GPU where there is one) against the
reference's own tools, on random databases written by the reference's `count` (needs oracle/_ref/jellyfish).
    python scripts/fuzz_readers.py [N] [SEED]
"""
import os
import random
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import jfutil  # noqa: E402

n_iter = int(sys.argv[1]) if len(sys.argv) > 1 else 50
rng = random.Random(int(sys.argv[2]) if len(sys.argv) > 2 else 1)


def rand_fasta(path, total):
    out = []
    for r in range(rng.randrange(1, 5)):
        n = rng.choice([50, 500, total])
        s = "".join(rng.choice("ACGT") for _ in range(n))
        if rng.random() < 0.4:
            s = s[:40] * (n // 40 + 1)
        out.append(">r%d\n%s\n" % (r, s))
    open(path, "w").write("".join(out))


def both(args, stdin=None):
    a = subprocess.run([jfutil.REF_JF] + args, stdout=subprocess.PIPE, stderr=subprocess.PIPE, input=stdin)
    b = subprocess.run([jfutil.OUR_JF] + args, stdout=subprocess.PIPE, stderr=subprocess.PIPE, input=stdin)
    return a, b


bad = 0


def report(it, what, args):
    global bad
    bad += 1
    print("MISMATCH #%d %s: %s" % (it, what, " ".join(args)))


with tempfile.TemporaryDirectory() as d:
    for it in range(n_iter):
        k = rng.choice([1, 3, 4, 8, 12, 16, 17, 21, 31, 32, 33, 47, 63, 64])
        size = rng.choice(["1k", "20k", "300k"])
        cargs = ["-m", str(k), "-s", size] + (["-C"] if rng.random() < 0.6 else []) + \
                (["--out-counter-len", str(rng.choice([1, 2, 3, 5]))] if rng.random() < 0.4 else [])
        fas, dbs = [], []
        for j in range(2):
            fa = os.path.join(d, "f%d_%d.fa" % (it, j))
            rand_fasta(fa, rng.choice([2000, 30000]))
            db = os.path.join(d, "db%d_%d.jf" % (it, j))
            subprocess.run([jfutil.REF_JF, "count", "-t", "2"] + cargs + ["-o", db, fa], check=True)
            fas.append(fa)
            dbs.append(db)
        db = dbs[0]
        # dump
        for _ in range(3):
            a = ["dump"] + rng.sample(["-c", "-t"], rng.randrange(0, 3)) + \
                (["-L", str(rng.choice([1, 2, 5, 300]))] if rng.random() < 0.4 else []) + \
                (["-U", str(rng.choice([1, 3, 50, 100000]))] if rng.random() < 0.4 else []) + [db]
            x, y = both(a)
            if x.returncode != y.returncode or x.stdout != y.stdout:
                report(it, "dump", a)
        # histo
        for _ in range(3):
            a = ["histo"] + (["-l", str(rng.choice([0, 1, 2, 10]))] if rng.random() < 0.5 else []) + \
                (["-h", str(rng.choice([1, 5, 100, 100000]))] if rng.random() < 0.5 else []) + \
                (["-i", str(rng.choice([1, 2, 7]))] if rng.random() < 0.4 else []) + (["-f"] if rng.random() < 0.3 else []) + [db]
            x, y = both(a)
            if x.returncode != y.returncode or x.stdout != y.stdout:
                report(it, "histo", a)
        # stats
        for _ in range(2):
            a = ["stats"] + (["-L", str(rng.choice([1, 2, 5]))] if rng.random() < 0.4 else []) + \
                (["-U", str(rng.choice([1, 3, 1000]))] if rng.random() < 0.4 else []) + [db]
            x, y = both(a)
            if x.returncode != y.returncode or x.stdout != y.stdout:
                report(it, "stats", a)
        # query: k-mers of the input, random k-mers, lower case, one with an N (both must treat it alike)
        seq = "".join(l.strip() for l in open(fas[0]) if not l.startswith(">"))
        mers = [seq[p:p + k] for p in (rng.randrange(0, max(1, len(seq) - k)) for _ in range(5)) if len(seq) >= k]
        mers += ["".join(rng.choice("ACGT") for _ in range(k)) for _ in range(3)]
        mers += [m.lower() for m in mers[:2]]
        a = ["query", db] + mers
        x, y = both(a)
        if x.returncode != y.returncode or x.stdout != y.stdout:
            report(it, "query", a)
        a = ["query", "-s", fas[1], db]
        x, y = both(a)
        if x.returncode != y.returncode or x.stdout != y.stdout:
            report(it, "query -s", a)
        # merge (same -m/-s => same matrix)
        ma, mb = os.path.join(d, "ma.jf"), os.path.join(d, "mb.jf")
        extra = (["-L", str(rng.choice([0, 1, 2, 3]))] if rng.random() < 0.3 else []) + (["-U", str(rng.choice([2, 100]))] if rng.random() < 0.3 else [])
        extra += rng.choice([[], [], ["-m"], ["--max"]])
        x = subprocess.run([jfutil.REF_JF, "merge", "-o", ma] + extra + dbs, stdout=subprocess.PIPE, stderr=subprocess.PIPE)
        y = subprocess.run([jfutil.OUR_JF, "merge", "-o", mb] + extra + dbs, stdout=subprocess.PIPE, stderr=subprocess.PIPE)
        if x.returncode != y.returncode:
            report(it, "merge exit %d/%d %s | %s" % (x.returncode, y.returncode, x.stderr[-100:], y.stderr[-100:]), extra + dbs)
        elif x.returncode == 0:
            h1, b1 = jfutil.split_db(ma)
            h2, b2 = jfutil.split_db(mb)
            if jfutil.semantic(h1) != jfutil.semantic(h2) or b1 != b2:
                report(it, "merge output", extra + dbs)
        # jaccard (two text lines instead of a database), three inputs
        ja, jb = os.path.join(d, "ja.txt"), os.path.join(d, "jb.txt")
        three = dbs + [dbs[0]] if rng.random() < 0.5 else dbs
        x = subprocess.run([jfutil.REF_JF, "merge", "-j", "-o", ja] + three, stdout=subprocess.PIPE, stderr=subprocess.PIPE)
        y = subprocess.run([jfutil.OUR_JF, "merge", "-j", "-o", jb] + three, stdout=subprocess.PIPE, stderr=subprocess.PIPE)
        if x.returncode != y.returncode or (x.returncode == 0 and open(ja, "rb").read() != open(jb, "rb").read()):
            report(it, "merge --jaccard", three)
        # text/sorted databases of the same inputs, merged as text
        tdbs = []
        for j in range(2):
            t = os.path.join(d, "t%d_%d.jf" % (it, j))
            subprocess.run([jfutil.REF_JF, "count", "-t", "2"] + [c for c in cargs if c not in ("--out-counter-len",)][:4 + ("-C" in cargs)] + ["--text", "-o", t, fas[j]], check=True)
            tdbs.append(t)
        x = subprocess.run([jfutil.REF_JF, "merge", "-o", ma] + extra + tdbs, stdout=subprocess.PIPE, stderr=subprocess.PIPE)
        y = subprocess.run([jfutil.OUR_JF, "merge", "-o", mb] + extra + tdbs, stdout=subprocess.PIPE, stderr=subprocess.PIPE)
        if x.returncode != y.returncode:
            report(it, "text merge exit %d/%d %s | %s" % (x.returncode, y.returncode, x.stderr[-100:], y.stderr[-100:]), extra + tdbs)
        elif x.returncode == 0:
            h1, b1 = jfutil.split_db(ma)
            h2, b2 = jfutil.split_db(mb)
            if jfutil.semantic(h1) != jfutil.semantic(h2) or b1 != b2:
                report(it, "text merge output", extra + tdbs)
        if bad:
            keep = "/tmp/fuzz_readers_fail"
            os.makedirs(keep, exist_ok=True)
            for f in fas + dbs:
                subprocess.run(["cp", f, keep])
            print("   count", " ".join(cargs), "(files kept in %s)" % keep)
            break
print("%d iterations, %d mismatches" % (it + 1, bad))
sys.exit(1 if bad else 0)
