"""What `count --sam` costs on the GPU.

1. Synthetic 150-bp reads as SAM lines with realistic fields (FLAG 0/4/16/256, CIGAR, tags), ~2 GB resident in HBM, counted at
   k = 21 -C from device memory; alternating with the same reads as FASTQ through the FASTQ path.  Whole-count k-mers/s from
   CUDA-synchronised wall time.
2. A separate profiled SAM count (torch.profiler): time of the transcode kernels (jf_sam.cu) next to the extraction kernel.
3. `count --sam` on a BGZF-compressed BAM file (read into pinned buffers by the CLI): wall time, and the time of the inflate
   alone (`inputs --sam`, the same reader, to /dev/null).

    python scripts/sam_bench.py [--gb 2] [--reps 3] [--bam-reads 400000] [--out FILE]

The result is one JSON line on standard output; --out also writes it, indented, to FILE.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

READ = 150
FLAGS = (b"0", b"4", b"16", b"256")


def make_reads(n, seed):
    rng = np.random.default_rng(seed)
    seq = np.frombuffer(b"ACGT", np.uint8)[rng.integers(0, 4, (n, READ))]
    qual = rng.integers(35, 74, (n, READ), dtype=np.uint8)
    return seq, qual


def sam_lines(seq, qual):
    """fixed-width SAM lines: every FLAG variant padded through QNAME to one width"""
    n = seq.shape[0]
    parts = []
    for flag in FLAGS:
        unm = flag == b"4"
        pre = b"\t".join([b"read_" + b"x" * (4 - len(flag)), flag, b"*" if unm else b"chr1", b"0" if unm else b"1234567",
                          b"0" if unm else b"60", b"*" if unm else b"150M", b"*", b"0", b"0", b""])
        parts.append(pre)
    w = max(len(p) for p in parts)
    parts = [p[:5] + b"y" * (w - len(p)) + p[5:] for p in parts]
    tail = b"\tNM:i:1\tMD:Z:75A74\tAS:i:145\tRG:Z:grp1\n"
    width = w + READ + 1 + READ + len(tail)
    out = np.empty((n, width), np.uint8)
    pre = np.stack([np.frombuffer(p, np.uint8) for p in parts])
    out[:, :w] = pre[np.arange(n) % 4]
    out[:, w:w + READ] = seq
    out[:, w + READ] = ord("\t")
    out[:, w + READ + 1:w + 2 * READ + 1] = qual
    out[:, w + 2 * READ + 1:] = np.frombuffer(tail, np.uint8)
    return b"@HD\tVN:1.6\tSO:unsorted\n@SQ\tSN:chr1\tLN:248956422\n", out.reshape(-1)


def fastq_records(seq, qual):
    n = seq.shape[0]
    head = b"@read_xxxxxxxx\n"
    width = len(head) + READ + 3 + READ + 1
    out = np.empty((n, width), np.uint8)
    out[:, :len(head)] = np.frombuffer(head, np.uint8)
    c = len(head)
    out[:, c:c + READ] = seq
    out[:, c + READ:c + READ + 3] = np.frombuffer(b"\n+\n", np.uint8)
    out[:, c + READ + 3:c + 2 * READ + 3] = qual
    out[:, -1] = ord("\n")
    return out.reshape(-1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gb", type=float, default=2.0)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--bam-reads", type=int, default=400000)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    from jellyfish_b200 import HashCounter
    import jfutil
    import sam_tools
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         stdout=subprocess.PIPE, text=True).stdout.strip().splitlines()[0]
    res = {"gpu": gpu}
    # ---- 1. device-resident SAM vs FASTQ ------------------------------------------------------------------------------
    line_bytes = 400
    n = int(a.gb * 1e9 / line_bytes)
    seq, qual = make_reads(n, 1)
    hdr, body = sam_lines(seq, qual)
    sam = torch.empty(len(hdr) + body.size, dtype=torch.uint8, device="cuda")
    sam[:len(hdr)] = torch.frombuffer(bytearray(hdr), dtype=torch.uint8).cuda()
    sam[len(hdr):] = torch.from_numpy(body).cuda()
    fq = torch.from_numpy(fastq_records(seq, qual)).cuda()
    del body, seq, qual
    kmers = n * (READ - 21 + 1)
    res.update({"reads": n, "sam_bytes": sam.numel(), "fastq_bytes": fq.numel(), "kmers": kmers})

    def run(t, is_sam):
        with HashCounter(1 << 31, 7, k=21, canonical=True) as hc:
            hc.add_device_text(fq[:1 << 20].data_ptr(), 1 << 20)       # (first launches and the record pool set up outside the window)
            hc.clear()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            hc.add_device_text(t.data_ptr(), t.numel(), sam=is_sam)
            st = hc.done()
            torch.cuda.synchronize()
            dt = time.perf_counter() - t0
            assert st["kmers"] == kmers, (st["kmers"], kmers)
            return dt, st["distinct"]
    times = {"sam": [], "fastq": []}
    distinct = {}
    for _ in range(a.reps):
        for name, t in (("sam", sam), ("fastq", fq)):
            dt, d = run(t, name == "sam")
            times[name].append(dt)
            distinct[name] = d
    assert distinct["sam"] == distinct["fastq"]
    for name in times:
        best = min(times[name])
        res[name] = {"seconds": times[name], "best_s": best, "kmers_per_s": kmers / best}
    # ---- 2. kernel times, profiled in a run of its own -----------------------------------------------------------------
    from torch.profiler import profile, ProfilerActivity
    with profile(activities=[ProfilerActivity.CUDA]) as p:
        run(sam, True)
    k = {}
    for ev in p.key_averages():
        nm = ev.key
        grp = "transcode" if "jfsam" in nm else "extract" if "extract_kernel" in nm else "other"
        k[grp] = k.get(grp, 0.0) + ev.device_time_total / 1e6
    res["kernels_s"] = k
    res["transcode_GBps_in"] = sam.numel() / k.get("transcode", float("nan")) / 1e9
    del sam, fq
    torch.cuda.empty_cache()
    # ---- 3. a BAM file through the CLI ---------------------------------------------------------------------------------
    with tempfile.TemporaryDirectory() as d:
        s2, q2 = make_reads(a.bam_reads, 2)
        h2, b2 = sam_lines(s2, q2)
        bam = sam_tools.bgzf(sam_tools.sam_to_bam(h2 + b2.tobytes()))
        path = os.path.join(d, "reads.bam")
        with open(path, "wb") as f:
            f.write(bam)
        t0 = time.perf_counter()
        subprocess.run([jfutil.OUR_JF, "inputs", "--sam", path], stdout=subprocess.DEVNULL, check=True)
        t_inflate = time.perf_counter() - t0
        t0 = time.perf_counter()
        subprocess.run([jfutil.OUR_JF, "count", "-m", "21", "-s", "256M", "-C", "--no-write", "-o", os.path.join(d, "x.jf"), "--sam", path], check=True)
        t_count = time.perf_counter() - t0
        res["bam"] = {"reads": a.bam_reads, "bgzf_bytes": len(bam), "count_wall_s": t_count, "inflate_only_s": t_inflate,
                      "inflate_share": t_inflate / t_count}
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
