#!/usr/bin/env python
"""Throughput of counting k-mers longer than 64 bases (k = 100 by default: four-word keys, the wide slot form, direct
insertion by K1) on one GPU, and of the reference on a bounded sample.

  * text: jfgpu_synth_fasta_device (seed 1) resident in HBM, counted with -C into a table sized for a load of about 0.5
    (2^l slots for about 2^(l-1) distinct k-mers); every step clears the table and counts the whole text again;
  * reported: k-mers/s over the timed steps (host clock around work that ends in a device synchronise), the kernel time of
    K1 from jfgpu_stats (seconds_count_kernel), the table's bytes, and the card's name and power limit;
  * reference: oracle/_ref/jellyfish count -t <cores> -m K -C on the first --sample-mbp Mbp of the same text, the
    Counting phase of --timing.

    python scripts/large_k_bench.py [--k 100] [--mbp 256] [--steps 3] [--sample-mbp 4]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import jfutil  # noqa: E402
from jellyfish_b200 import HashCounter  # noqa: E402
from jellyfish_b200 import _lib as L  # noqa: E402


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       stdout=subprocess.PIPE, stderr=subprocess.PIPE, universal_newlines=True)
    name, power, clk = [x.strip() for x in q.stdout.splitlines()[0].split(",")]
    return {"gpu": name, "power_limit": power, "max_sm_clock": clk}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--k", type=int, default=100)
    ap.add_argument("--mbp", type=int, default=256, help="Mbp of text per step")
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--sample-mbp", type=int, default=4, help="Mbp the reference counts")
    a = ap.parse_args()
    import torch
    lib = L.load()
    n_bases = a.mbp * 1000000
    nb = lib.jfgpu_synth_fasta_bytes(n_bases)
    text = torch.empty(nb + 16, dtype=torch.uint8, device="cuda")
    got = C.c_uint64(0)
    if lib.jfgpu_synth_fasta_device(0, C.c_void_p(text.data_ptr()), nb, n_bases, 1, C.byref(got), None):
        raise RuntimeError("jfgpu_synth_fasta_device failed")
    torch.cuda.synchronize()
    size = 1
    while size < 2 * n_bases:
        size <<= 1
    res = dict(gpu_info(), k=a.k, canonical=True, bases_per_step=n_bases)
    with HashCounter(size, 7, k=a.k, canonical=True) as hc:
        hc.add_device_text(text.data_ptr(), got.value)          # warm-up
        hc.done()
        info = hc.info()
        times, kern = [], []
        for _ in range(a.steps):
            hc.clear()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            hc.add_device_text(text.data_ptr(), got.value)
            st = hc.done()
            times.append(time.perf_counter() - t0)
            kern.append(st["seconds_count_kernel"])
        res.update(table_slots=info["size"], slot_bits=info["slot_bits"], table_bytes=info["table_bytes"],
                   distinct=st["distinct"], load=st["distinct"] / info["size"], kmers=st["kmers"], regrows=st["regrows"],
                   step_s=sorted(times), kmers_per_s=st["kmers"] / sorted(times)[len(times) // 2],
                   k1_kernel_s=sorted(kern))
        sample = text[:min(got.value, a.sample_mbp * 1000000 * 71 // 70 + 8)].cpu().numpy().tobytes()
    if os.path.exists(jfutil.REF_JF):
        with tempfile.TemporaryDirectory() as d:
            fa = os.path.join(d, "sample.fa")
            with open(fa, "wb") as f:
                f.write(sample[:sample.rfind(b"\n") + 1])
            tm = os.path.join(d, "timing")
            cores = os.cpu_count()
            jfutil.run([jfutil.REF_JF, "count", "-t", str(cores), "-m", str(a.k), "-C", "-s", str(4 * a.sample_mbp * 1000000),
                        "--timing", tm, "-o", os.path.join(d, "ref.jf"), fa])
            secs = float([line.split()[1] for line in open(tm) if line.startswith("Counting")][0])
            n_k = a.sample_mbp * 1000000 - a.k + 1
            res["reference"] = {"threads": cores, "bases": a.sample_mbp * 1000000, "counting_s": secs, "kmers_per_s": n_k / secs}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
