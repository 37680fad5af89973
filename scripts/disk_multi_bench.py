"""Cost of `count_multi --disk`: spills and the CPU merge, next to the same count with a table that never fills.

    python scripts/disk_multi_bench.py [--mbp 100] [--seed 11] [--worlds 1,2,4,8] [--out results.json]

A FASTA file of `--mbp` million random bases (seed `--seed`, 70-column lines) is written to a temporary directory and
counted with k = 21, canonical, at every world size the machine has GPUs for (the others are reported as not run):
- `--disk` with -s SPILL_SIZE: 2^25 slots for 1e8 distinct 21-mers, so each rank spills about three times;
- the same count with -s NOSPILL_SIZE (2^28), which never fills.
Per rank the script reports the spills, the seconds inside the spill hook (dump and write of the pieces) and the seconds
of the merge, which count_multi prints on stderr, and per run the wall time of the command.  The two outputs must have the
same records (their matrices differ, so the bodies are compared by an order-independent digest).  One JSON line per run, and the
GPU's name and power limit, go to stdout and to --out.
"""
import argparse
import json
import os
import re
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SPILL_SIZE, NOSPILL_SIZE = 1 << 25, 1 << 28


def write_fasta(path, n_bases, seed):
    rs = np.random.RandomState(seed)
    acgt = np.frombuffer(b"ACGT", np.uint8)
    with open(path, "wb") as f:
        f.write(b">bench\n")
        step = 70 * (1 << 16)
        for off in range(0, n_bases, step):
            m = min(step, n_bases - off)
            seq = acgt[rs.randint(0, 4, size=m)]
            full = m // 70 * 70
            lines = np.concatenate([seq[:full].reshape(-1, 70), np.full((full // 70, 1), 10, np.uint8)], axis=1).tobytes()
            f.write(lines)
            if m > full:
                f.write(seq[full:].tobytes() + b"\n")


def run(world, size, disk, fa, out, port):
    args = ["-m", "21", "-s", str(size), "-C", "-o", out, fa] + (["--disk"] if disk else [])
    mod = ["-m", "jellyfish_b200.count_multi"]
    cmd = [sys.executable] + mod + args if world == 1 else \
        [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(world), "--master-addr", "127.0.0.1",
         "--master-port", str(port)] + mod + args
    env = dict(os.environ, SOURCE_DATE_EPOCH="0")
    for v in ("RANK", "WORLD_SIZE", "LOCAL_RANK"):
        env.pop(v, None)
    t0 = time.perf_counter()
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, cwd=ROOT, env=env)
    wall = time.perf_counter() - t0
    log = r.stdout.decode(errors="replace")
    if r.returncode:
        raise SystemExit("count_multi failed:\n" + log[-3000:])
    ranks = {}
    for m in re.finditer(r"rank (\d+) --disk: spills (\d+) spill_s ([\d.]+) merge_s ([\d.]+)", log):
        ranks[int(m.group(1))] = {"spills": int(m.group(2)), "spill_s": float(m.group(3)), "merge_s": float(m.group(4))}
    return wall, [ranks[r] for r in sorted(ranks)]


def digest(path):
    """(records, an order-independent sum over them): the two outputs have different matrices, so their record orders differ"""
    with open(path, "rb") as f:
        hlen = int(f.read(9))
        h = json.loads(f.read(hlen).rstrip(b"\0"))
        rec = (h["key_len"] + 7) // 8 + h["counter_len"]
        n, total = 0, 0
        mult = np.array([0x9E3779B97F4A7C15, 0xC2B2AE3D27D4EB4F], np.uint64)
        while True:
            data = f.read(rec << 22)
            if not data:
                break
            body = np.frombuffer(data, np.uint8).reshape(-1, rec)
            wide = np.zeros((len(body), 16), np.uint8)
            wide[:, :rec] = body
            w = wide.view(np.uint64) * mult
            total = (total + int(np.bitwise_xor(w[:, 0], w[:, 1] >> np.uint64(7)).sum(dtype=np.uint64))) & ((1 << 64) - 1)
            n += len(body)
    return n, total


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mbp", type=int, default=100)
    ap.add_argument("--seed", type=int, default=11)
    ap.add_argument("--worlds", default="1,2,4,8")
    ap.add_argument("--out")
    a = ap.parse_args()
    import torch
    n_gpu = torch.cuda.device_count()
    if n_gpu == 0:
        raise SystemExit("no GPU: nothing measured")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], stdout=subprocess.PIPE,
                         text=True).stdout.strip().splitlines()
    results = [{"gpus": gpu, "mbp": a.mbp, "seed": a.seed, "k": 21, "spill_size": SPILL_SIZE, "nospill_size": NOSPILL_SIZE}]
    with tempfile.TemporaryDirectory() as d:
        fa = os.path.join(d, "bench.fa")
        write_fasta(fa, a.mbp * 1000000, a.seed)
        for i, world in enumerate(int(w) for w in a.worlds.split(",")):
            if world > n_gpu:
                results.append({"world": world, "not_run": "only %d GPU(s)" % n_gpu})
                continue
            wall_d, ranks = run(world, SPILL_SIZE, True, fa, os.path.join(d, "disk.jf"), 29400 + 10 * i)
            wall_n, _ = run(world, NOSPILL_SIZE, False, fa, os.path.join(d, "plain.jf"), 29405 + 10 * i)
            same = digest(os.path.join(d, "disk.jf")) == digest(os.path.join(d, "plain.jf"))
            results.append({"world": world, "disk_wall_s": round(wall_d, 3), "nospill_wall_s": round(wall_n, 3), "ranks": ranks,
                            "same_records": same})
            for p in ("disk.jf", "plain.jf"):
                os.unlink(os.path.join(d, p))
            print(json.dumps(results[-1]), flush=True)
    print(json.dumps(results[0]))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
