"""Time `count_multi` on one input file split among the ranks (`--split auto`) against the same text cut into N files, one
per rank (`--split files`).

    python scripts/split_bench.py [--worlds 1,2,4,8] [--k 31] [--gbp-per-gpu 1.25] [--dir DIR] [--out FILE]

For each world N it writes one synthetic FASTA on local disk (one '>read1' record, 70-column lines, iid ACGT from a seeded
numpy generator, `--gbp-per-gpu` x N bases) and the same bases cut at line ends into N files (each its own '>read1'
record, so k-1 fewer k-mers per extra file), reads every file once (the page cache is warm for every timed run: this
script changes no system setting, so a cold cache is not measured), then runs `count_multi` under torchrun (plain python
for N = 1) once per mode.  The issue's sizes are 1.25 Gbp per GPU at k = 31 and 5 Gbp per GPU at k = 21 (`--k 21
--gbp-per-gpu 5`; -s is sized for the distinct k-mers).

Reported per world and mode: wall time of the whole command (process start, NCCL set-up, table allocation, the count and
the dump included), k-mers per second over that time, and the read rate (input bytes over that time).  With a warm cache
the read rate is memory bandwidth, not the disk's.  The GPU's name, power limit and SM clocks are read in the same run.
Prints one JSON line; --out also writes it to a file.
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
LINE = 70


def write_fasta(paths, n_bases, seed):
    """n_bases of iid ACGT in 70-column lines, cut at line ends into len(paths) files of one record each.  Line j's bases
    depend only on (seed, j), so every cut gives the same text."""
    lut = np.frombuffer(b"ACGT", np.uint8)
    n_lines = (n_bases + LINE - 1) // LINE
    per = [(n_lines * i // len(paths), n_lines * (i + 1) // len(paths)) for i in range(len(paths))]
    block = 1 << 20                                        # lines per generated block

    def rows(q):
        b0, b1 = q * block, min(n_lines, (q + 1) * block)
        r = np.empty((b1 - b0, LINE + 1), np.uint8)
        r[:, :LINE] = lut[np.random.default_rng([seed, q]).integers(0, 4, (b1 - b0, LINE), dtype=np.uint8)]
        r[:, LINE] = 10
        return b0, r
    for path, (l0, l1) in zip(paths, per):
        with open(path, "wb") as f:
            f.write(b">read1\n")
            for q in range(l0 // block, (l1 + block - 1) // block):
                b0, r = rows(q)
                first = max(l0, b0)
                r = r[first - b0:min(l1, b0 + len(r)) - b0]
                data = r.reshape(-1)
                if first + len(r) == n_lines and n_bases % LINE and len(r):       # the file's last line is short
                    data = np.concatenate((data[:-(LINE + 1)], r[-1, :n_bases % LINE], [10])).astype(np.uint8)
                f.write(data.tobytes())


def warm(paths):
    for p in paths:
        with open(p, "rb") as f:
            while f.read(64 << 20):
                pass


def run(world, args, port):
    env = dict(os.environ, SOURCE_DATE_EPOCH="0")
    cmd = [sys.executable, "-m"] if world == 1 else [sys.executable, "-m", "torch.distributed.run", "--nnodes=1",
                                                     "--nproc-per-node", str(world), "--master-addr", "127.0.0.1",
                                                     "--master-port", str(port), "-m"]
    t0 = time.perf_counter()
    r = subprocess.run(cmd + ["jellyfish_b200.count_multi"] + args, cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
    dt = time.perf_counter() - t0
    if r.returncode:
        raise SystemExit(r.stdout.decode(errors="replace")[-3000:])
    return dt


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                           stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else None
    except (OSError, subprocess.SubprocessError):
        return None


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--worlds", default="1,2,4,8")
    ap.add_argument("--k", type=int, default=31)
    ap.add_argument("--gbp-per-gpu", type=float, default=1.25)
    ap.add_argument("--dir", default=None, help="local disk for the inputs (default: a temporary directory)")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    n_dev = torch.cuda.device_count()
    if n_dev == 0:
        raise SystemExit("split_bench: no CUDA device")
    worlds = [w for w in (int(x) for x in a.worlds.split(",")) if w <= n_dev]
    res = {"bench": "split", "k": a.k, "gbp_per_gpu": a.gbp_per_gpu, "gpu": gpu_info(), "page_cache": "warm", "runs": []}
    with tempfile.TemporaryDirectory(dir=a.dir) as d:
        for world in worlds:
            n_bases = int(a.gbp_per_gpu * 1e9) * world
            one = os.path.join(d, "one.fa")
            parts = [os.path.join(d, "part%d.fa" % i) for i in range(world)]
            write_fasta([one], n_bases, seed=world)
            write_fasta(parts, n_bases, seed=world)
            nbytes = os.path.getsize(one)
            size = 1 << max(20, int(np.ceil(np.log2(n_bases * 1.25))))       # a table for ~n_bases distinct k-mers
            base = ["-m", str(a.k), "-s", str(size), "-C", "-o", os.path.join(d, "out.jf")]
            for mode, files in (("auto", [one]), ("files", parts)):
                warm(files)
                dt = run(world, base + ["--split", mode] + files, 29700 + world)
                kmers = n_bases - len(files) * (a.k - 1)
                res["runs"].append({"world": world, "split": mode, "n_files": len(files), "bytes": nbytes, "wall_s": round(dt, 3),
                                    "kmers_per_s": kmers / dt, "read_GBps": nbytes / dt / 1e9})
                for f in os.listdir(d):
                    if f.startswith("out.jf"):
                        os.unlink(os.path.join(d, f))
            for p in [one] + parts:
                os.unlink(p)
    res["gpu_after"] = gpu_info()
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
