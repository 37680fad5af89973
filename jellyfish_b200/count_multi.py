"""`jellyfish count` over several GPUs of one node.

    torchrun --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 -m jellyfish_b200.count_multi \
        -m 21 -s 16G -C -o mer_counts.jf reads_1.fa reads_2.fa ...

Every rank parses the files `files[rank::N]` (a file is the unit of distribution: no k-mer spans two
files, mer_overlap_sequence_parser.hpp:111), the k-mers are routed to the rank that owns their table
position, each rank writes `OUT.<rank>`, and rank 0 concatenates the shards in rank order into OUT --
byte-identical to what one GPU (or the reference) writes for the same input, since shard r holds
exactly the positions r*size/N ... (r+1)*size/N - 1.  (`jellyfish merge` on the shard files gives the
same records: jellyfish/merge_files.cc:45-176.)  -m takes 1..128; k > 64 (32-byte keys) is routed by the key exchange
on 2, 4 or 8 GPUs, with 64 MB batches.

Bloom structures (k <= 64) take the key exchange: `--bc FILE` is loaded whole by every rank and tested before a k-mer is
routed; `--bf-size N` (the GLOBAL expected number of k-mers) gives every rank a filter for its share, applied by the
owner after the exchange, where every occurrence of a k-mer arrives.
"""
import argparse
import os
import sys

import torch
import torch.distributed as dist

from .distributed import ShardedCounter, concat_shards


def _size(v):
    mult = {"k": 10**3, "M": 10**6, "G": 10**9, "T": 10**12}
    return int(v[:-1]) * mult[v[-1]] if v[-1] in mult else int(v)


def main(argv=None):
    ap = argparse.ArgumentParser(prog="jellyfish_b200.count_multi", description=__doc__.split("\n")[0])
    ap.add_argument("-m", "--mer-len", type=int, required=True)
    ap.add_argument("-s", "--size", type=_size, required=True, help="GLOBAL table size (as for jellyfish count)")
    ap.add_argument("-C", "--canonical", action="store_true")
    ap.add_argument("-c", "--counter-len", type=int, default=7)
    ap.add_argument("-p", "--reprobes", type=int, default=126)
    ap.add_argument("--out-counter-len", type=int, default=4)
    ap.add_argument("-L", "--lower-count", type=int, default=0)
    ap.add_argument("-U", "--upper-count", type=int, default=(1 << 64) - 1)
    ap.add_argument("-o", "--output", default="mer_counts.jf")
    ap.add_argument("--bf-size", type=_size, default=0, help="Bloom prefilter: expected number of k-mers (GLOBAL)")
    ap.add_argument("--bf-fp", type=float, default=0.01, help="false positive rate of the Bloom prefilter")
    ap.add_argument("--bc", help="count only the k-mers this Bloom counter (written by `bc`) holds twice")
    ap.add_argument("--keep-shards", action="store_true")
    ap.add_argument("files", nargs="+")
    a = ap.parse_args(argv)
    # the single-GPU command's checks (count_main.cc:196-197 and the k <= 64 scope of every Bloom structure)
    if a.bf_size and a.bc:
        sys.stderr.write("Error: Switches [--bf-size] and [--bc] conflict\n")
        sys.exit(1)
    if a.mer_len > 64 and (a.bf_size or a.bc):
        sys.stderr.write("Error: --bf-size and --bc take mer lengths up to 64\n")
        sys.exit(1)

    rank, world = int(os.environ.get("RANK", "0")), int(os.environ.get("WORLD_SIZE", "1"))
    local = int(os.environ.get("LOCAL_RANK", rank))
    torch.cuda.set_device(local)
    if world > 1:
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        os.environ.setdefault("NCCL_MAX_CTAS", "16")      # K1 leaves 16 SMs to the exchange that runs beside it
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    sc = ShardedCounter(a.size, a.counter_len, k=a.mer_len, canonical=a.canonical, rank=rank, world=world, device=local,
                        reprobes=a.reprobes, bf_size=a.bf_size, bf_fp=a.bf_fp, bc=a.bc)
    mine = a.files[rank::world]
    rounds = torch.tensor([len(mine)], device="cuda")
    if world > 1:
        dist.all_reduce(rounds, op=dist.ReduceOp.MAX)       # every rank takes part in every exchange
    for i in range(int(rounds.item())):
        if i < len(mine):
            with open(mine[i], "rb") as f:
                data = f.read()
            if data[:1] not in (b">", b"@", b""):
                raise SystemExit("Unsupported format: %s" % mine[i])
            buf = torch.zeros(max(16, len(data) + 256), dtype=torch.uint8, device="cuda")
            if data:
                buf[:len(data)] = torch.frombuffer(bytearray(data), dtype=torch.uint8).cuda()
            sc.add_device_text(buf.data_ptr(), len(data))
            del buf
        else:
            sc.add_device_text(0, 0)
    st = sc.done()
    cmdline = ["count_multi"] + (argv if argv is not None else sys.argv[1:])
    sc.hc.dump("%s.%d" % (a.output, rank), lower=a.lower_count, upper=a.upper_count, out_counter_len=a.out_counter_len, cmdline=cmdline)
    if world > 1:
        dist.barrier()
    if rank == 0:
        concat_shards(a.output, world, a.output)
        if not a.keep_shards:
            for r in range(world):
                os.unlink("%s.%d" % (a.output, r))
        sys.stderr.write("count_multi: %d GPUs, %d k-mers on rank 0's share, output %s\n" % (world, st["kmers"], a.output))
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
