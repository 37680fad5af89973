"""The single-GPU steps bench.py measures, at full size, checked against an exact sort-based count (tests/kmer_model.py).

For every config of bench.CONFIGS without a Bloom prefilter, the text bench.py generates for rank 0 (text A) and for rank 1
(text B) is counted by the model first, with only the text resident.  The engine is then created as bench.py creates it
(default record pool, batch size and regions) and runs the bench's step: clear(), the whole text from device memory,
done().  After each step the statistics, the count histogram and the counts of 65 536 sampled input k-mers and of about as
many random keys (nearly all absent) must equal the model's.

  step 1  a fresh engine, text A
  step 2  clear(), text B.  The whole dump is streamed through kmer_model.StreamDigest: every partition's digest must be
          model B's and (original position, key) must strictly increase.  As every digest holds the number of distinct
          keys and the sum of their hashes, no key of text A may survive the clear.
  step 3  (k21) clear(), text B fed from pinned host memory (the bench's e2e path, 64 MB host batches), checked as step 2.

Engines as bench.py creates them (table_setup / part_configure):
  k21  -s 8G: lsize 33, 32-bit slots (34 GB), 1024 regions of 2^23 slots, 4-byte records: the window form of K2
  k31  -s 2G: lsize 31, 64-bit slots (17 GB), 256 regions of 2^23 slots, 8-byte records
  k63  -s 2G: lsize 31, 128-bit slots (34 GB), 512 regions of 2^22 slots, 16-byte records

On a mismatch the first partition that differs is recounted alone and its keys are looked up in the engine; up to 20 wrong
keys are printed with their original position, region and window."""
import ctypes as C
import json
import time

import numpy as np
import pytest

import jfutil
import kmer_model as km

pytestmark = pytest.mark.gpu

import bench                                                       # noqa: E402  (the configs and seeds the bench runs)

CONFIGS = [name for name, cfg in bench.CONFIGS.items() if not cfg["bf"]]
SEEDS = [(0x9E3779B97F4A7C15 * (rank + 1)) & ((1 << 64) - 1) for rank in (0, 1)]       # bench.py, ranks 0 and 1
EXPECT = {"k21": (33, 32, 1024, 4), "k31": (31, 64, 256, 8), "k63": (31, 128, 512, 16)}  # lsize, slot_bits, regions, record bytes
N_RANDOM = 70_000
UINT64_MAX = (1 << 64) - 1


def _synth(lib, text, n_bases, seed):
    import torch
    got = C.c_uint64(0)
    rc = lib.jfgpu_synth_fasta_device(0, C.c_void_p(text.data_ptr()), text.numel(), n_bases, seed, C.byref(got), None)
    assert rc == 0, "synthetic FASTA generation failed"
    torch.cuda.synchronize()
    return got.value


def _queries(text, k, n_bases):
    """65 536 input k-mers at bench.py's seeded sample positions, then N_RANDOM random canonical keys."""
    import torch
    starts = np.random.default_rng(bench.SAMPLE_SEED).integers(0, n_bases - k + 1, size=bench.SAMPLE_KMERS, dtype=np.int64)
    base = torch.from_numpy(starts[:, None] + np.arange(k, dtype=np.int64)[None, :]).cuda()
    sampled = km.mers_words(text[7 + base + base // 70], k)         # base i sits at byte 7 + i + i // 70
    return torch.cat([sampled, km.random_words(N_RANDOM, k, 4242, "cuda")])


def _lookup(hc, words, piece=1 << 16):
    """Engine counts of (n, W) keys through jfgpu_lookup, in slices of numpy arrays."""
    arr = np.ascontiguousarray(words.cpu().numpy()).view(np.uint64).reshape(-1)
    n, W = words.shape
    vals = np.zeros(n, np.uint64)
    for a in range(0, n, piece):
        m = min(piece, n - a)
        hc._check(hc._lib.jfgpu_lookup(hc._h, C.c_void_p(arr[a * W:].ctypes.data), m, C.c_void_p(vals[a:].ctypes.data)))
    return vals.astype(np.int64)


def _dump_digest(hc, info, k, P):
    """Stream the whole dump (4-byte counts) through a StreamDigest; every slice is read from the engine's pinned buffer in
    place and digested on the GPU."""
    import torch
    from jellyfish_b200 import _lib
    assert not info["matrix_identity"]
    sd = km.StreamDigest(k, info["size"], info["matrix_columns"], 4, P, "cuda")
    err = []

    def sink(ctx, ptr, n):
        try:
            sd.feed_address(ptr, n)
            return 0
        except BaseException as e:           # (an exception cannot cross the C frame)
            err.append(e)
            return 1
    cb = _lib.SINK_FN(sink)
    nrec = C.c_uint64(0)
    rc = hc._lib.jfgpu_dump(hc._h, 0, UINT64_MAX, 4, cb, None, C.byref(nrec))
    if err:
        raise err[0]
    hc._check(rc)
    sd.finish()
    torch.cuda.empty_cache()
    assert sd.n_records == nrec.value
    return sd


def _diagnose(hc, text, k, info, model, p):
    """Recount partition p alone and look its keys up in the engine -> lines describing up to 20 wrong keys."""
    import torch
    lines = []
    try:
        torch.cuda.empty_cache()
        uniq, counts = km.partition_counts(text, k, model.P, p, chunk_bases=1 << 24)
        got = _lookup(hc, uniq, piece=1 << 20)
        want = counts.cpu().numpy()
        bad = np.nonzero(got != want)[0]
        lines.append("partition %d: %d keys, %d with a wrong engine count" % (p, len(want), len(bad)))
        if len(bad):
            sd = km.StreamDigest(k, info["size"], info["matrix_columns"], 4, model.P, "cuda")
            w = uniq[torch.from_numpy(bad[:20]).cuda()]
            a = torch.stack([km._shr(w[:, b // 8], 8 * (b % 8)) & 255 if b % 8 else w[:, b // 8] & 255
                             for b in range(sd.kb)], 1)
            pos = sd.positions(a).tolist()
            rbits = info["lsize"] - (info["part_regions"].bit_length() - 1) if info["part_regions"] else None
            for i, row in enumerate(w.tolist()):
                key = sum((x & UINT64_MAX) << (64 * j) for j, x in enumerate(row))
                lines.append("  key %#x: model %d, engine %d, position %d, region %s, window %d"
                             % (key, want[bad[i]], got[bad[i]], pos[i], pos[i] >> rbits if rbits else "-", pos[i] >> 14))
        del uniq, counts
    except Exception as e:                    # the diagnosis must not hide the mismatch it explains
        lines.append("diagnosis of partition %d failed: %r" % (p, e))
    return "\n".join(lines)


def _check_step(hc, st, text, k, info, model, queries, what):
    assert st["kmers"] == model.n_kmers, (what, st["kmers"], model.n_kmers)
    assert st["inserted"] == st["kmers"], (what, st)
    assert st["distinct"] == model.distinct(), (what, st["distinct"], model.distinct())
    hist = hc.histogram(km.N_BINS)
    if hist != model.histogram():
        first = [(i, a, b) for i, (a, b) in enumerate(zip(hist, model.histogram())) if a != b][:10]
        raise AssertionError("%s: histogram differs (bin, engine, model): %s" % (what, first))
    got = _lookup(hc, queries)
    want = model.query_counts.numpy()
    bad = np.nonzero(got != want)[0]
    if len(bad):
        parts = km.partition_of(km.key_hash(queries[torch_index(bad[:1])]), model.P).tolist()
        raise AssertionError("%s: %d of %d lookups differ, first at query %d (engine %d, model %d)\n%s"
                             % (what, len(bad), len(want), bad[0], got[bad[0]], want[bad[0]],
                                _diagnose(hc, text, k, info, model, parts[0])))


def _check_dump(hc, text, k, info, model, what):
    sd = _dump_digest(hc, info, k, model.P)
    diff = km.differing_partitions(model, sd)
    msg = ""
    if diff or sd.n_disorder:
        p = diff[0] if diff else 0
        msg = ("%s: %d records (model %d distinct keys), %d out of (position, key) order (first: %s), partitions that differ: %s\n"
               "partition %d digest engine %s model %s\n%s"
               % (what, sd.n_records, model.distinct(), sd.n_disorder, sd.first_disorder, diff[:20], p,
                  sd.digest[p].tolist(), model.digest[p].tolist(), _diagnose(hc, text, k, info, model, p)))
    assert not diff and sd.n_disorder == 0 and sd.n_records == model.distinct(), msg


def torch_index(a):
    import torch
    return torch.from_numpy(np.asarray(a, dtype=np.int64)).cuda()


@pytest.mark.parametrize("name", CONFIGS)
def test_bench_step_is_exact_at_full_size(name, built):
    import torch
    from jellyfish_b200 import HashCounter, _lib
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    cfg = bench.CONFIGS[name]
    k, n_bases, size = cfg["k"], cfg["bases"], bench.parse_size(cfg["size"])
    torch.cuda.set_device(0)
    total = torch.cuda.get_device_properties(0).total_memory
    if total < 80e9:
        pytest.skip("the bench's %s configuration needs an 80 GB device (this one has %.1f GB)" % (name, total / 1e9))
    lib = _lib.load()
    nbytes = lib.jfgpu_synth_fasta_bytes(n_bases)
    geo = jfutil.geometry(k, (size - 1).bit_length())
    table_bytes = (1 << geo["lsize"]) * geo["slot_bits"] // 8
    free = torch.cuda.mem_get_info(0)[0]
    if free < nbytes + table_bytes + (8 << 30):
        pytest.skip("the bench's %s configuration needs %.1f GB free (text, table, 8 GB of pool), %.1f GB are"
                    % (name, (nbytes + table_bytes + (8 << 30)) / 1e9, free / 1e9))
    t_all = time.perf_counter()
    times = {}

    # ---- the models, with only the text resident ----
    text = torch.empty(nbytes + 256, dtype=torch.uint8, device="cuda")
    models, queries = [], []
    for seed in SEEDS:
        n_text = _synth(lib, text, n_bases, seed)
        q = _queries(text, k, n_bases)
        torch.cuda.reset_peak_memory_stats()
        t0 = time.perf_counter()
        models.append(km.count(text[:n_text], k, queries=q))
        times.setdefault("model_s", []).append(time.perf_counter() - t0)
        times.setdefault("model_peak_gb", []).append(torch.cuda.max_memory_allocated() / 1e9)
        queries.append(q)
        assert models[-1].n_kmers == n_bases - k + 1
        assert (models[-1].query_counts[:bench.SAMPLE_KMERS] > 0).all()
        assert (models[-1].query_counts[bench.SAMPLE_KMERS:] == 0).sum() >= bench.SAMPLE_KMERS
    del q
    torch.cuda.empty_cache()
    times["P"] = models[0].P
    model_a, model_b = models

    # ---- the engine as bench.py creates it ----
    n_text = _synth(lib, text, n_bases, SEEDS[0])
    hc = HashCounter(size, 7, k=k, canonical=True, device=0, bf_size=0)
    try:
        info = hc.info()
        assert (info["lsize"], info["slot_bits"], info["part_regions"], info["part_rec_bytes"]) == EXPECT[name], info

        # step 1: fresh engine, text A
        t0 = time.perf_counter()
        hc.clear()
        hc.add_device_text(text.data_ptr(), n_text)
        st = hc.done()
        times["step_s"] = time.perf_counter() - t0
        times["free_gb_after_step"] = torch.cuda.mem_get_info(0)[0] / 1e9
        _check_step(hc, st, text[:n_text], k, info, model_a, queries[0], "%s step 1 (text A)" % name)

        # step 2: clear, text B; then the whole dump
        n_text = _synth(lib, text, n_bases, SEEDS[1])
        hc.clear()
        hc.add_device_text(text.data_ptr(), n_text)
        st = hc.done()
        _check_step(hc, st, text[:n_text], k, info, model_b, queries[1], "%s step 2 (clear, text B)" % name)
        t0 = time.perf_counter()
        _check_dump(hc, text[:n_text], k, info, model_b, "%s step 2 dump" % name)
        times["dump_s"] = time.perf_counter() - t0

        # step 3 (k21): clear, text B from pinned host memory
        if name == "k21":
            hptr = lib.jfgpu_host_alloc(n_text)
            assert hptr, "pinned host allocation failed"
            try:
                host = torch.frombuffer((C.c_uint8 * n_text).from_address(hptr), dtype=torch.uint8)
                host.copy_(text[:n_text])
                torch.cuda.synchronize()
                hc.clear()
                hc.add_text((C.c_void_p(hptr), n_text))
                st = hc.done()
                del host
            finally:
                lib.jfgpu_host_free(hptr)
            _check_step(hc, st, text[:n_text], k, info, model_b, queries[1], "%s step 3 (clear, text B from host memory)" % name)
            _check_dump(hc, text[:n_text], k, info, model_b, "%s step 3 dump" % name)
    finally:
        hc.close()
        del text
        torch.cuda.empty_cache()
    times["wall_s"] = time.perf_counter() - t_all
    print("bench_exact %s %s" % (name, json.dumps(times)))
