#!/usr/bin/env python
"""Regenerate tests/golden/golden_query.json from the UNMODIFIED reference (oracle/_ref/jellyfish, built by
`make -C oracle all` where the reference sources are present).

`query -s` of the inputs of tests/gen.py against databases the reference's `count` wrote.  Per database: the `count`
switches and inputs, its header keys, body md5 and `histo` output; per query: the database, the `-s` files, the md5 and
the line count of the standard output.  tests/test_gpu_query.py rebuilds every database with `jellyfish-b200 count`
and runs `jellyfish-b200 query -s` on the GPU against these.
    python scripts/make_query_golden.py
"""
import json
import os
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import gen  # noqa: E402
import jfutil  # noqa: E402

DBS = {
    "k17C": (["-m", "17", "-s", "1M", "-C"], ["multi.fa"]),
    "k31": (["-m", "31", "-s", "1M"], ["plain.fa", "multi.fa"]),
    "k40C": (["-m", "40", "-s", "1M", "-C"], ["plain.fa", "multi.fa"]),
    "k5": (["-m", "5", "-s", "1k"], ["multi.fa"]),                                  # table as large as the key space
    "k21_ocl1": (["-m", "21", "-s", "1M", "--out-counter-len", "1"], ["polya.fa", "repeat.fa"]),   # clipped counts
}
# (the '\r' that ends the reference's 4096-byte parser buffer is left out: DESIGN.md section 7a)
QUERIES = [[f] for f in ("plain.fa", "dos.fa", "noeol.fa", "lower.fa", "multi.fa", "multi2.fa", "one_per_line.fa",
                         "blank_runs.fa", "long_header.fa", "reads.fq", "reads_dos.fq", "empty.fa", "header_only.fa")]
QUERIES.append(["plain.fa", "reads.fq", "multi2.fa", "empty.fa", "dos.fa"])                # several -s files in one call


def main():
    out = {"dbs": {}, "queries": []}
    with tempfile.TemporaryDirectory() as d:
        inputs = gen.make_all(d)
        for name, (args, ins) in DBS.items():
            db = os.path.join(d, name + ".jf")
            jfutil.run([jfutil.REF_JF, "count", "-t", "1"] + args + ["-o", db] + [inputs[i] for i in ins])
            h, b = jfutil.split_db(db)
            out["dbs"][name] = {"args": args, "inputs": ins, "header": jfutil.semantic(h), "body_md5": jfutil.md5(b),
                                "histo": jfutil.run([jfutil.REF_JF, "histo", db]).stdout.decode()}
            for files in QUERIES:
                cmd = [jfutil.REF_JF, "query"] + sum([["-s", inputs[f]] for f in files], []) + [db]
                so = jfutil.run(cmd).stdout
                out["queries"].append({"db": name, "files": files, "md5": jfutil.md5(so), "lines": so.count(b"\n")})
    path = os.path.join(ROOT, "tests", "golden", "golden_query.json")
    with open(path, "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")
    print("wrote %s: %d databases, %d queries" % (path, len(out["dbs"]), len(out["queries"])))


if __name__ == "__main__":
    main()
