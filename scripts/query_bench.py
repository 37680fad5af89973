#!/usr/bin/env python
"""Throughput of `query -s` on the GPU: load a database into a table, then look up every k-mer of a text in input order.

One call, one JSON line on standard output:
  * the card's name and power limit (nvidia-smi);
  * count 1 Gbp of jfgpu_synth_fasta_device text (seed 1) at k=21 -C; its records go to host memory;
  * load those records into a fresh table (jfgpu_load_records): records/s;
  * query 2 Gbp of pinned host text, 1 Gbp of it the database's own text (seed 1) and 1 Gbp new text (seed 2), with a
    sink that discards the lines, after a warm-up query: k-mers/s and output GB/s;
  * the CPU yardstick: oracle/_ref/jellyfish query -s (the reference binary build() makes) and jellyfish-b200 query -s on
    a 20 Mbp sample against a database of 20 Mbp; both outputs must be equal, and two device runs byte-identical.
    python scripts/query_bench.py [--gbp 1] [--sample-mbp 20]
"""
import argparse
import ctypes as C
import hashlib
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402

import jfutil  # noqa: E402
from jellyfish_b200 import HashCounter  # noqa: E402
from jellyfish_b200 import _lib as L  # noqa: E402


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       stdout=subprocess.PIPE, stderr=subprocess.PIPE, universal_newlines=True)
    name, power, clk = [x.strip() for x in q.stdout.splitlines()[0].split(",")]
    return {"gpu": name, "power_limit": power, "max_sm_clock": clk}


def synth_host(lib, n_bases, seed):
    """jfgpu_synth_fasta_device text of n_bases, copied to pinned host memory -> (pointer, size)."""
    import torch
    nb = lib.jfgpu_synth_fasta_bytes(n_bases)
    dev = torch.empty(nb, dtype=torch.uint8, device="cuda")
    got = C.c_uint64(0)
    if lib.jfgpu_synth_fasta_device(0, C.c_void_p(dev.data_ptr()), nb, n_bases, seed, C.byref(got), None):
        raise RuntimeError("jfgpu_synth_fasta_device failed")
    torch.cuda.synchronize()
    host = lib.jfgpu_host_alloc(got.value)
    if not host:
        raise RuntimeError("pinned allocation of %d bytes failed" % got.value)
    text = dev.cpu().numpy()                  # (kept alive until the copy is done)
    C.memmove(host, text.ctypes.data, got.value)
    return host, got.value


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gbp", type=float, default=1.0, help="Gbp counted into the database (the query reads twice as much)")
    ap.add_argument("--sample-mbp", type=int, default=20)
    a = ap.parse_args()
    lib = L.load()
    res = dict(gpu_info(), k=21, canonical=True)
    nbp = int(a.gbp * 1e9)

    # the database: count, then its records in host memory
    db_txt, db_n = synth_host(lib, nbp, 1)
    with HashCounter(2 * nbp, k=21, canonical=True) as hc:
        hc.add_text((db_txt, db_n))
        st = hc.done()
        n_rec = st["distinct"]
        recs = np.empty(n_rec * ((2 * 21 + 7) // 8 + 4), dtype=np.uint8)     # 6 key bytes, 4 count bytes
        at = [0]

        def keep(chunk):
            recs[at[0]:at[0] + len(chunk)] = np.frombuffer(chunk, dtype=np.uint8)
            at[0] += len(chunk)
        hc.dump_records(out_counter_len=4, sink=keep)
    assert at[0] == len(recs)
    res.update(db_bases=nbp, db_records=n_rec, db_bytes=int(recs.nbytes))

    with HashCounter(2 * n_rec, k=21, canonical=True) as hc:
        t0 = time.perf_counter()
        hc.load_records((recs.ctypes.data, recs.nbytes), 4)
        hc.done()
        t_load = time.perf_counter() - t0
        res.update(load_s=round(t_load, 4), load_records_per_s=round(n_rec / t_load, 1), load_regrows=hc.stats()["regrows"])
        del recs
        # query: the database's own text, then new text (two files)
        q2_txt, q2_n = synth_host(lib, nbp, 2)
        warm = min(db_n, 64 << 20)
        hc.query_text((db_txt, warm), sink="discard")
        t0 = time.perf_counter()
        lines = hc.query_text((db_txt, db_n), sink="discard")
        out_b = hc.query_bytes
        lines += hc.query_text((q2_txt, q2_n), sink="discard")
        out_b += hc.query_bytes
        t_q = time.perf_counter() - t0
        res.update(query_bases=2 * nbp, query_kmers=lines, query_s=round(t_q, 4),
                   query_kmers_per_s=round(lines / t_q, 1), query_output_bytes=out_b,
                   query_output_GB_per_s=round(out_b / t_q / 1e9, 3))
    lib.jfgpu_host_free(db_txt)
    lib.jfgpu_host_free(q2_txt)

    # CPU yardstick on a sample (files on disk, both binaries through their command line)
    with tempfile.TemporaryDirectory() as d:
        sb = a.sample_mbp * 1000000
        paths = {}
        for name, n, seed in (("db.fa", sb, 1), ("q1.fa", sb // 2, 1), ("q2.fa", sb - sb // 2, 3)):
            p, nbytes = synth_host(lib, n, seed)
            paths[name] = os.path.join(d, name)
            with open(paths[name], "wb") as f:
                f.write(C.string_at(p, nbytes))
            lib.jfgpu_host_free(p)
        db = os.path.join(d, "sample.jf")
        jfutil.run([jfutil.OUR_JF, "count", "-m", "21", "-s", str(2 * sb), "-C", "-o", db, paths["db.fa"]])
        qargs = ["query", "-s", paths["q1.fa"], "-s", paths["q2.fa"], db]
        md5s = []
        for _ in range(2):
            t0 = time.perf_counter()
            out = jfutil.run([jfutil.OUR_JF] + qargs).stdout
            t_dev = time.perf_counter() - t0
            md5s.append(hashlib.md5(out).hexdigest())
        res.update(sample_bases=sb, sample_kmers=out.count(b"\n"), sample_device_cli_s=round(t_dev, 3),
                   sample_two_runs_identical=md5s[0] == md5s[1])
        if os.path.exists(jfutil.REF_JF):
            t0 = time.perf_counter()
            ref = jfutil.run([jfutil.REF_JF] + qargs).stdout
            t_ref = time.perf_counter() - t0
            res.update(sample_reference_cli_s=round(t_ref, 3), sample_reference_kmers_per_s=round(ref.count(b"\n") / t_ref, 1),
                       sample_equal_to_reference=hashlib.md5(ref).hexdigest() == md5s[0])
        else:
            res.update(sample_reference_cli_s=None)
    print(json.dumps(res, sort_keys=True))


if __name__ == "__main__":
    main()
