#!/usr/bin/env python
"""Bloom structures on the sharded path, on one GPU and, where there are several, over all of them.

  * one GPU: --gbp Gbp of jfgpu_synth_fasta_device text (seed 1) resident in HBM, k = 21 -C, as rank 0 of a world of
    --world shards (global table of --world * 2^--shard-log2 slots), text in batches of 256 MB as count_multi takes it:
      - route: jfgpu_extract_route without and with a loaded Bloom counter (count --bc; a counter of m = 14 * --bc-kmers
        positions with random digits); routed k-mers/s over the whole text;
      - insert: jfgpu_insert_keys of rank 0's own bucket of one batch, without and with the owner-side --bf-size filter
        (sized for the text's k-mers), straight into the table and staged region by region (part_min_mb = 1); keys/s;
      - fold: jfgpu_bloom_fold of one counter into another, both of --fold-kmers k-mers at -f 0.001; GB/s of counter words;
    each the median over --steps timed steps after one warm-up, host clock around work that ends in a device synchronise;
  * with >= 2 GPUs: `torchrun -m jellyfish_b200.count_multi --bf-size` on --gbp-per-gpu Gbp of synthetic text per GPU
    (one file per rank, weak scaling); wall time of the command and k-mers/s per GPU.
The card's name, power limit and maximum SM clock come from nvidia-smi in the same call.  One JSON line.

    python scripts/shard_bloom_bench.py [--gbp 1] [--steps 3] [--world 8] [--shard-log2 28]
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
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from jellyfish_b200 import BloomCounter, HashCounter  # noqa: E402
from jellyfish_b200 import _lib as L  # noqa: E402
from large_k_shard_bench import gpu_info, synth, timed  # noqa: E402

BATCH = 256 << 20


def median(t):
    return t[len(t) // 2]


def one_gpu(a, lib, res):
    import numpy as np
    import torch
    text, n = synth(lib, int(a.gbp * 1e9), 1)
    world, k = a.world, 21
    cap = BATCH // world * 5 // 4 + 65536
    keys = torch.empty((world, cap), dtype=torch.int64, device="cuda")
    counts = torch.zeros(world, dtype=torch.int64, device="cuda")
    eng = dict(k=k, canonical=True, shard_index=0, n_shards=world, allow_regrow=False, max_batch_bytes=BATCH)

    def route_all(hc):
        routed = 0
        for off in range(0, n, BATCH):
            ln = min(BATCH, n - off)
            counts.zero_()
            hc.extract_route(text.data_ptr() + off, ln, keys.data_ptr(), cap, counts.data_ptr(), begin=off == 0, end=off + ln >= n)
            routed += int(counts.sum().item())
        return routed

    res["route"] = {"world": world}
    with HashCounter(world << a.shard_log2, 7, **eng) as hc:
        t = timed(a.steps, lambda: route_all(hc))
        routed = route_all(hc)
        res["route"]["plain"] = {"kmers": routed, "step_s": t, "kmers_per_s": routed / median(t)}
        m = 14 * a.bc_kmers
        body = np.random.default_rng(3).integers(0, 243, size=(m + 4) // 5, dtype=np.uint8).tobytes()
        cols = (C.c_uint64 * (2 * k))(*[(0x9E3779B97F4A7C15 * (i + 1)) & ((1 << 64) - 1) for i in range(2 * k)])
        cols2 = (C.c_uint64 * (2 * k))(*[(0xC2B2AE3D27D4EB4F * (i + 3)) & ((1 << 64) - 1) for i in range(2 * k)])
        hc._check(lib.jfgpu_bloom_load(hc._h, m, 10, cols, cols2, body, len(body)))
        t = timed(a.steps, lambda: route_all(hc))
        kept = route_all(hc)
        res["route"]["bc"] = {"m": m, "kmers_in": routed, "kmers_kept": kept, "step_s": t, "kmers_per_s": routed / median(t)}
    # rank 0's own bucket of the first batch
    with HashCounter(world << a.shard_log2, 7, **eng) as hc:
        counts.zero_()
        hc.extract_route(text.data_ptr(), min(BATCH, n), keys.data_ptr(), cap, counts.data_ptr())
        own = int(counts[0].item())
    res["insert"] = {"keys": own, "local_slots": 1 << a.shard_log2}
    for name, bf, part in (("direct", 0, {"no_partition": True}), ("direct_bf", n, {"no_partition": True}),
                           ("staged", 0, {"part_min_mb": 1}), ("staged_bf", n, {"part_min_mb": 1})):
        with HashCounter(world << a.shard_log2, 7, bf_size=bf, **dict(eng, **part)) as hc:
            def insert():
                hc.insert_keys(keys[0].data_ptr(), own)
                hc.done()
            t = timed(a.steps, insert, before=hc.clear)
            st = hc.done()
            res["insert"][name] = {"regions": hc.info()["part_regions"], "inserted": st["inserted"], "step_s": t,
                                   "keys_per_s": own / median(t)}
    del keys, counts, text
    torch.cuda.empty_cache()
    with BloomCounter(a.fold_kmers, 0.001, k=k, canonical=True) as x, BloomCounter(a.fold_kmers, 0.001, k=k, canonical=True) as y:
        _, nw = x.words()
        py, _ = y.words()
        t = timed(a.steps, lambda: x.fold(py, 0, nw))
        res["fold"] = {"m": x.info()["m"], "words": nw, "step_s": t, "counter_gb_per_s": nw * 4 / median(t) / 1e9}


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
               "127.0.0.1", "--master-port", "29671", "-m", "jellyfish_b200.count_multi", "-m", "21", "-C",
               "-s", str(world << a.shard_log2), "--bf-size", str(world * n_bases), "-o", out] + files
        t0 = time.perf_counter()
        r = subprocess.run(cmd, cwd=ROOT, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, universal_newlines=True)
        wall = time.perf_counter() - t0
        if r.returncode:
            res["multi"] = {"world": world, "error": r.stdout[-2000:]}
            return
        kmers = world * (n_bases - 20)
        res["multi"] = {"world": world, "bases_per_gpu": n_bases, "wall_s": wall, "kmers_per_s_per_gpu": kmers / wall / world}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gbp", type=float, default=1.0, help="Gbp of text on one GPU")
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--world", type=int, default=8, help="shards of the one-GPU measurements")
    ap.add_argument("--shard-log2", type=int, default=28, help="log2 of the slots of one shard")
    ap.add_argument("--bc-kmers", type=int, default=1 << 28, help="k-mers the loaded counter is sized for")
    ap.add_argument("--fold-kmers", type=int, default=1 << 30, help="k-mers the folded counters are sized for")
    ap.add_argument("--gbp-per-gpu", type=float, default=1.0, help="Gbp of text per GPU of the multi-GPU run")
    ap.add_argument("--world-multi", type=int, default=8, help="GPUs of the multi-GPU run at most")
    ap.add_argument("--tmp", default=None, help="directory for the multi-GPU input files")
    a = ap.parse_args()
    import torch
    lib = L.load()
    res = dict(gpu_info(), k=21, canonical=True, bases=int(a.gbp * 1e9))
    one_gpu(a, lib, res)
    ngpu = torch.cuda.device_count()
    res["multi"] = "not measured: %d GPU" % ngpu
    if ngpu >= 2:
        multi_gpu(a, lib, ngpu, res)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
