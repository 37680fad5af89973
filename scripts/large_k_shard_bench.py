#!/usr/bin/env python
"""Sharded counting of k-mers longer than 64 bases (four-word keys, the key exchange), on one GPU and, where there are
several, over all of them.

  * one GPU: --mbp Mbp of jfgpu_synth_fasta_device text (seed 1) resident in HBM, k = 100 -C:
      - route: jfgpu_extract_route as rank 0 of a world of --world shards (global table of --world * 2^--shard-log2 slots),
        every bucket large enough for the whole text; routed k-mers/s;
      - insert: jfgpu_insert_keys of rank 0's own bucket into its shard of 2^--shard-log2 wide slots (cleared every step);
        keys/s;
      - direct: what scripts/large_k_bench.py measures, the same text counted by direct insertion (K1 claims and publishes
        wide slots itself) into a single table at load about 0.5; k-mers/s;
    each the median over --steps timed steps after one warm-up, host clock around work that ends in a device synchronise;
  * with >= 2 GPUs: `torchrun -m jellyfish_b200.count_multi` on --gbp-per-gpu Gbp of synthetic text per GPU (one file per
    rank, weak scaling) into --world-multi * 2^--shard-log2 slots; wall time of the command and k-mers/s per GPU.
The card's name, power limit and maximum SM clock come from nvidia-smi in the same call.  One JSON line.

    python scripts/large_k_shard_bench.py [--mbp 256] [--steps 3] [--world 8] [--shard-log2 29]
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
from jellyfish_b200 import HashCounter  # noqa: E402
from jellyfish_b200 import _lib as L  # noqa: E402


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       stdout=subprocess.PIPE, stderr=subprocess.PIPE, universal_newlines=True)
    name, power, clk = [x.strip() for x in q.stdout.splitlines()[0].split(",")]
    return {"gpu": name, "power_limit": power, "max_sm_clock": clk}


def synth(lib, n_bases, seed, device=0):
    import torch
    nb = lib.jfgpu_synth_fasta_bytes(n_bases)
    text = torch.empty(nb + 16, dtype=torch.uint8, device="cuda:%d" % device)
    got = C.c_uint64(0)
    if lib.jfgpu_synth_fasta_device(device, C.c_void_p(text.data_ptr()), nb, n_bases, seed, C.byref(got), None):
        raise RuntimeError("jfgpu_synth_fasta_device failed")
    torch.cuda.synchronize()
    return text, got.value


def timed(steps, fn, before=None):
    import torch
    fn()                                     # warm-up
    times = []
    for _ in range(steps):
        if before:
            before()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        times.append(time.perf_counter() - t0)
    return sorted(times)


def one_gpu(a, lib, res):
    import torch
    text, n = synth(lib, a.mbp * 1000000, 1)
    k = a.k
    world = a.world
    # route buckets that hold the whole text whatever the split (k-mers <= bases)
    cap = (a.mbp * 1000000 // world) * 5 // 4 + (1 << 20)
    keys = torch.empty((world, cap * 4), dtype=torch.int64, device="cuda")
    counts = torch.zeros(world, dtype=torch.int64, device="cuda")
    with HashCounter(world << a.shard_log2, 7, k=k, canonical=True, shard_index=0, n_shards=world, allow_regrow=False) as hc:
        def route():
            hc.extract_route(text.data_ptr(), n, keys.data_ptr(), cap, counts.data_ptr())
        t_route = timed(a.steps, route, before=counts.zero_)
        c = counts.tolist()
        routed = sum(c)
        own = c[0]

        def insert():
            hc.insert_keys(keys[0].data_ptr(), own)
            hc.done()
        t_ins = timed(a.steps, insert, before=hc.clear)
        st = hc.done()
        info = hc.info()
        res["route"] = {"world": world, "kmers": routed, "step_s": t_route, "kmers_per_s": routed / t_route[len(t_route) // 2],
                        "bucket_max_over_mean": max(c) / (routed / world)}
        res["insert"] = {"keys": own, "local_slots": 1 << a.shard_log2, "table_bytes": info["table_bytes"],
                         "distinct": st["distinct"], "load": st["distinct"] / (1 << a.shard_log2), "step_s": t_ins,
                         "keys_per_s": own / t_ins[len(t_ins) // 2]}
    del keys, counts
    torch.cuda.empty_cache()
    size = 1
    while size < 2 * a.mbp * 1000000:
        size <<= 1
    with HashCounter(size, 7, k=k, canonical=True) as hc:
        def direct():
            hc.add_device_text(text.data_ptr(), n)
            hc.done()
        t_dir = timed(a.steps, direct, before=hc.clear)
        st = hc.done()
        res["direct"] = {"table_slots": size, "distinct": st["distinct"], "load": st["distinct"] / size, "kmers": st["kmers"],
                         "step_s": t_dir, "kmers_per_s": st["kmers"] / t_dir[len(t_dir) // 2]}
    res["route_over_direct"] = res["route"]["kmers_per_s"] / res["direct"]["kmers_per_s"]


def multi_gpu(a, lib, ngpu, res):
    import torch
    world = min(ngpu, a.world_multi)
    n_bases = int(a.gbp_per_gpu * 1e9)
    with tempfile.TemporaryDirectory(dir=a.tmp) as d:
        files = []
        for r in range(world):
            text, n = synth(lib, n_bases, 100 + r)
            p = os.path.join(d, "r%d.fa" % r)
            text[:n].cpu().numpy().tofile(p)
            files.append(p)
            del text
        torch.cuda.empty_cache()
        out = os.path.join(d, "out.jf")
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(world), "--master-addr",
               "127.0.0.1", "--master-port", "29651", "-m", "jellyfish_b200.count_multi", "-m", str(a.k), "-C",
               "-s", str(world << a.shard_log2_multi), "-o", out] + files
        t0 = time.perf_counter()
        r = subprocess.run(cmd, cwd=ROOT, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, universal_newlines=True)
        wall = time.perf_counter() - t0
        if r.returncode:
            res["multi"] = {"world": world, "error": r.stdout[-2000:]}
            return
        kmers = world * (n_bases - a.k + 1)
        res["multi"] = {"world": world, "bases_per_gpu": n_bases, "slots": world << a.shard_log2_multi, "wall_s": wall,
                        "kmers_per_s_per_gpu": kmers / wall / world, "db_bytes": os.path.getsize(out)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--k", type=int, default=100)
    ap.add_argument("--mbp", type=int, default=256, help="Mbp of text on one GPU")
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--world", type=int, default=8, help="shards of the one-GPU route / insert measurement")
    ap.add_argument("--shard-log2", type=int, default=29, help="log2 of the wide slots of one shard (one GPU)")
    ap.add_argument("--gbp-per-gpu", type=float, default=1.0, help="Gbp of text per GPU of the multi-GPU run")
    ap.add_argument("--world-multi", type=int, default=8, help="GPUs of the multi-GPU run at most")
    ap.add_argument("--shard-log2-multi", type=int, default=30, help="log2 of the wide slots of one shard (multi-GPU)")
    ap.add_argument("--tmp", default=None, help="directory for the multi-GPU input files")
    a = ap.parse_args()
    import torch
    lib = L.load()
    res = dict(gpu_info(), k=a.k, canonical=True, bases=a.mbp * 1000000)
    one_gpu(a, lib, res)
    ngpu = torch.cuda.device_count()
    if ngpu >= 2:
        multi_gpu(a, lib, ngpu, res)
    else:
        res["multi"] = "not run: %d GPU" % ngpu
    print(json.dumps(res))


if __name__ == "__main__":
    main()
