"""List the kernels a build of libjfgpu.so launches on a fixed set of small scenarios (needs a GPU).

    python scripts/tools/launch_trace.py [LIB] > launches.txt

LIB defaults to the package's own library.  Each scenario runs under torch.profiler (CUDA activities); the listing gives,
per scenario, the number of launches the engine counted (jfgpu_kernel_launches) and then one line per kernel in launch
order: name, grid, block and shared memory (as the profiler reports it: static + dynamic bytes).  Two builds that make
the same launches print the same listing, so a host-side refactor is checked with `diff` of two listings.  The texts
are drawn from fixed seeds.

The scenarios cover the region-by-region paths: the window form of K2 at k2_mode 0, 3 and 4 and a second drain into a
table in memory, the L2 forms at k2_mode 1 and 2, a doubling in the middle of a write-only drain and in the L2 form, a
full spill list before the first drain, PRIME / UPDATE, routed keys staged by insert_keys, the record exchange
(shard_extract / pack / unpack), text fed from host and from device memory, query, and k = 63 in 128-bit slots.  They
also cover the calls that hold buffers of their own: dump, lookup and histogram at k = 21 and k = 100 (the wide
kernels), a database loaded with a doubling in the middle and then queried, count --bf-size, and a Bloom counter built,
dumped and loaded back in front of a table.
"""
import json
import os
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)


def fasta(n, seed, period=0):
    """n random bases (a repeat of `period` random bases when period > 0) as FASTA with lines of 70"""
    import numpy as np
    rng = np.random.default_rng(seed)
    base = np.frombuffer(b"ACGT", np.uint8)[rng.integers(0, 4, period or n)]
    seq = np.resize(base, n).tobytes()
    return b">r\n" + b"\n".join(seq[i:i + 70] for i in range(0, n, 70)) + b"\n"


def scenarios(tmp):
    import torch
    from jellyfish_b200 import BloomCounter, HashCounter, load_database
    from jellyfish_b200.distributed import CHUNK

    def win(**kw):            # k=17, 2^23 32-bit slots, 256 regions, 4-byte records: the window form under part_min_mb=1
        return HashCounter(8_000_000, 7, k=17, canonical=True, part_min_mb=1, pool_bytes=1 << 30, max_batch_bytes=1 << 20, **kw)

    def dev(data):
        buf = torch.zeros(len(data) + 256, dtype=torch.uint8, device="cuda")
        buf[:len(data)] = torch.frombuffer(bytearray(data), dtype=torch.uint8).cuda()
        return buf

    A, G = fasta(3_000_000, 501), fasta(9_500_000, 502)

    def window(mode):
        def run():
            with win(k2_mode=mode) as hc:
                hc.add_text(A); hc.done()
                hc.add_text(A); hc.done()               # the second drain finds the table in memory
        return run

    def l2(mode):
        def run():
            with win(k2_mode=mode) as hc:
                hc.add_text(A); hc.done()
        return run

    def lazy_regrow():
        with win() as hc:
            hc.add_text(A); hc.done(); hc.clear()
            hc.add_text(G); hc.done()

    def spill_list():
        with win() as hc:
            hc.add_text(fasta(1_000_000, 505) + fasta(30_000_000, 507, period=3)); hc.done()

    def l2_regrow():
        with HashCounter(1_000_000, 7, k=21, canonical=True, part_min_mb=1, max_batch_bytes=1 << 20) as hc:
            hc.add_text(fasta(4_000_000, 508)); hc.done()

    def prime_update():
        with HashCounter(1_000_000, 7, k=17, canonical=True, part_min_mb=1, pool_bytes=128 << 20, max_batch_bytes=1 << 20) as hc:
            hc.set_op(HashCounter.OP_PRIME); hc.add_text(fasta(500_000, 509))
            hc.set_op(HashCounter.OP_UPDATE); hc.add_text(A); hc.done()

    def device_text():
        buf = dev(A)
        with win() as hc:
            hc.add_device_text(buf.data_ptr(), len(A)); hc.done()

    def route_insert_keys():
        world, cap = 2, 400_000
        shards = [HashCounter(4_000_000, 7, k=21, canonical=True, shard_index=r, n_shards=world, allow_regrow=False,
                              max_batch_bytes=200_000, part_min_mb=1, pool_bytes=256 << 20) for r in range(world)]
        keys = torch.zeros((world, cap), dtype=torch.int64, device="cuda")
        counts = torch.zeros(world, dtype=torch.int64, device="cuda")
        data = fasta(600_000, 510)
        buf = dev(data)
        for off in range(0, len(data), 150_000):
            ln = min(150_000, len(data) - off)
            counts.zero_()
            torch.cuda.synchronize()
            shards[0].extract_route(buf.data_ptr() + off, ln, keys.data_ptr(), cap, counts.data_ptr(), begin=off == 0,
                                    end=off + ln >= len(data))
            for d, c in enumerate(counts.tolist()):
                shards[d].insert_keys(keys[d].data_ptr(), c)
        for hc in shards:
            hc.done(); hc.close()

    def record_exchange():
        world = 2
        n_sm = torch.cuda.get_device_properties(0).multi_processor_count
        arena = 2 * n_sm * (1024 // world) + 64
        shards, bufs = [], []
        for r in range(world):
            hc = HashCounter(4_000_000, 7, k=17, canonical=True, shard_index=r, n_shards=world, allow_regrow=False,
                             part_min_mb=1, pool_bytes=2 << 30, max_batch_bytes=1 << 20)
            b = [torch.empty(n, dtype=torch.uint8, device="cuda") for n in
                 (2 * world * arena * CHUNK, 2 * world * arena * 8, world * arena * CHUNK, world * arena * 8)]
            assert hc.shard_setup(b[0].data_ptr(), b[1].data_ptr(), arena, b[2].data_ptr(), b[3].data_ptr(), arena)
            shards.append(hc); bufs.append(b)
        data = fasta(500_000, 511)
        buf = dev(data)
        for n_round, off in enumerate(range(0, len(data), 170_000)):
            ln, bank = min(170_000, len(data) - off), n_round & 1
            shards[0].shard_extract(buf.data_ptr() + off, ln, bank, begin=off == 0, end=off + ln >= len(data))
            counts = shards[0].shard_pack(bank)
            for d in range(world):
                c, a0 = counts[d], (bank * world + d) * arena
                bufs[d][2][:c * CHUNK] = bufs[0][0][a0 * CHUNK:(a0 + c) * CHUNK]
                bufs[d][3][:c * 8] = bufs[0][1][a0 * 8:(a0 + c) * 8]
                torch.cuda.synchronize()
                shards[d].shard_unpack([c] + [0] * (world - 1))
                torch.cuda.synchronize()
        for hc in shards:
            hc.done(); hc.close()

    def query():
        with win() as hc:
            hc.add_text(A); hc.done()
            hc.query_text(fasta(200_000, 512))

    def k63_wide_slots():
        with HashCounter(2_000_000, 7, k=63, canonical=True, part_min_mb=1, max_batch_bytes=1 << 20) as hc:
            assert hc.info()["slot_bits"] == 128
            hc.add_text(fasta(1_000_000, 513)); hc.done()

    def dump_lookup_histogram(k):
        def run():
            with HashCounter(2_000_000, 7, k=k, canonical=True, max_batch_bytes=1 << 20) as hc:
                hc.add_text(fasta(1_000_000, 514)); hc.done()
                hc.dump_records(sink="discard")
                hc.get_many(list(range(1000)))
                hc.histogram()
        return run

    def database():
        """a k=21 database of about 900k distinct k-mers"""
        path = os.path.join(tmp, "db.jf")
        with HashCounter(4_000_000, 7, k=21, canonical=True, max_batch_bytes=1 << 20) as hc:
            hc.add_text(fasta(1_000_000, 515)); hc.done()
            hc.dump(path)
        return path

    def load_with_doubling():
        hc = load_database(database(), size=1 << 17, max_batch_bytes=1 << 20)      # the table doubles while it loads
        try:
            assert hc.info()["size"] > 1 << 17
        finally:
            hc.close()

    def query_database():
        hc = load_database(database(), max_batch_bytes=1 << 20)
        try:
            hc.query_text(fasta(300_000, 516))
        finally:
            hc.close()

    def bloom_filter():
        with HashCounter(2_000_000, 7, k=21, canonical=True, bf_size=2_000_000, max_batch_bytes=1 << 20) as hc:
            hc.add_text(fasta(1_000_000, 517)); hc.done()

    def bloom_counter():
        path = os.path.join(tmp, "bc.bin")
        with BloomCounter(2_000_000, k=21, canonical=True, max_batch_bytes=1 << 20) as bc:
            bc.add_text(fasta(1_000_000, 518))
            bc.dump(path)
        with HashCounter(2_000_000, 7, k=21, canonical=True, max_batch_bytes=1 << 20) as hc:
            hc.load_bloom_counter(path)
            hc.add_text(fasta(1_000_000, 518)); hc.done()

    return [("window_k2_mode_%d" % m, window(m)) for m in (0, 3, 4)] + [("l2_k2_mode_%d" % m, l2(m)) for m in (1, 2)] + [
        ("regrow_in_write_only_drain", lazy_regrow), ("full_spill_list", spill_list), ("regrow_l2_form", l2_regrow),
        ("prime_update", prime_update), ("device_text", device_text), ("route_insert_keys", route_insert_keys),
        ("record_exchange", record_exchange), ("query", query), ("k63_128bit_slots", k63_wide_slots),
        ("dump_lookup_histogram_k21", dump_lookup_histogram(21)), ("dump_lookup_histogram_k100", dump_lookup_histogram(100)),
        ("load_database_doubling", load_with_doubling), ("query_loaded_database", query_database),
        ("count_bf_size", bloom_filter), ("bloom_counter_dump_load", bloom_counter)]


def kernels(trace_path):
    with open(trace_path) as f:
        ev = json.load(f)["traceEvents"]
    ks = sorted((e for e in ev if e.get("cat") == "kernel"), key=lambda e: e["ts"])
    return ["%s grid=%s block=%s smem=%s" % (e["name"], e["args"].get("grid"), e["args"].get("block"), e["args"].get("shared memory"))
            for e in ks]


def main():
    from jellyfish_b200 import _lib
    if len(sys.argv) > 1:
        _lib.LIB_PATH = os.path.abspath(sys.argv[1])
    lib = _lib.load()
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.zeros(1, device="cuda")
    with tempfile.TemporaryDirectory() as d:
        for name, run in scenarios(d):
            torch.cuda.synchronize()
            n0 = lib.jfgpu_kernel_launches()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                run()
                torch.cuda.synchronize()
            n = lib.jfgpu_kernel_launches() - n0
            path = os.path.join(d, name + ".json")
            prof.export_chrome_trace(path)
            ks = kernels(path)
            print("## %s: %d engine launches, %d kernels traced" % (name, n, len(ks)))
            for k in ks:
                print(k)
            sys.stdout.flush()


if __name__ == "__main__":
    main()
