"""`jellyfish bc` over several GPUs of one node.

    torchrun --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 -m jellyfish_b200.bc_multi \
        -m 21 -s 5G -C -o reads.bc reads_1.fa reads_2.fa ...

Every rank builds a Bloom counter of its share of every file (`--split auto`, the default: the split of count_multi, with
the seam parsed through jfgpu_seam_host and the FASTQ cuts checked afterwards; a failed check clears every counter and
falls back to whole files; a path that is not a regular file is fed whole by one rank) or of the files `files[rank::N]` (`--split files`), with the same k, size and false positive rate, so every counter has the same m, number of hashes and matrices.  The counters
are folded into one, rank r holding slice r of it (a reduce-scatter in bounded pieces), every rank writes the bytes of
its slice to `OUT.<rank>`, and rank 0 writes the header and the slices in rank order into OUT -- byte-identical to what
one GPU (or the reference) writes for the same input, since a position of the counter ends at min(2, hits) whatever
the order of the hits (bloom_counter2.hpp:56-107).
"""
import argparse
import ctypes as C
import os
import sys

import torch
import torch.distributed as dist

import numpy as np

from .count_multi import _size
from .distributed import ShardedBloomCounter, ShareReader, concat_bloom_slices, fastq_cuts_agree
from .split import plan_file, splittable

PIECE = 64 << 20          # bytes of a share read and fed at a time


def add_split(sbc, files, rank, world, k):
    """Feed this rank's share of every regular file (anything else whole by rank i % world); False when a FASTQ share did
    not start on a record."""
    tallies = []
    for i, path in enumerate(files):
        if not splittable(path):
            if i % world == rank:
                sbc.add_files([path])         # (read once, from its start; the engine refuses what is not FASTA / FASTQ)
            continue
        try:
            share = plan_file(path, rank, world, k)
        except ValueError:
            raise SystemExit("Unsupported format: %s" % path)
        if share is None:
            continue
        reader = ShareReader(path, share, PIECE)
        newlines = 0
        try:
            seam = reader.seam()
            if seam:
                sbc.bc.seam_text(seam, fmt=share.fmt)
            for j in range(reader.n_pieces):
                hptr, n, begin, end = reader.read(j)
                reader.prefetch(j + 1)
                if share.fmt == "fastq":
                    newlines += int(np.count_nonzero(np.ctypeslib.as_array((C.c_uint8 * n).from_address(hptr)) == 10))
                sbc.bc.add_text((hptr, n), begin=begin, end=end, fmt=share.fmt)
                reader.release(j)
        finally:
            reader.close()
        if share.fmt == "fastq":
            tallies.append([share.end - share.start, newlines])
    return fastq_cuts_agree(tallies, world, "cuda")


def add_files(sbc, files, rank, world):
    for path in files[rank::world]:
        with open(path, "rb") as f:
            if f.read(1) not in (b">", b"@", b""):
                raise SystemExit("Unsupported format: %s" % path)
    sbc.add_files(files[rank::world])


def main(argv=None):
    ap = argparse.ArgumentParser(prog="jellyfish_b200.bc_multi", description=__doc__.split("\n")[0])
    ap.add_argument("-m", "--mer-len", type=int, required=True)
    ap.add_argument("-s", "--size", type=_size, required=True, help="expected number of k-mers (all ranks together)")
    ap.add_argument("-f", "--fpr", type=float, default=0.001, help="false positive rate")
    ap.add_argument("-C", "--canonical", action="store_true")
    ap.add_argument("-o", "--output", default="mer_counts.bc")
    ap.add_argument("--keep-shards", action="store_true")
    ap.add_argument("--split", choices=("auto", "files"), default="auto",
                    help="auto: split every file among the ranks; files: give rank r the whole files files[r::N]")
    ap.add_argument("files", nargs="+")
    a = ap.parse_args(argv)
    if a.mer_len < 1 or a.mer_len > 64:
        sys.stderr.write("Error: jellyfish-b200 bc supports mer lengths 1..64 (no Bloom counter for longer k-mers)\n")
        sys.exit(1)

    rank, world = int(os.environ.get("RANK", "0")), int(os.environ.get("WORLD_SIZE", "1"))
    local = int(os.environ.get("LOCAL_RANK", rank))
    torch.cuda.set_device(local)
    if world > 1:
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    sbc = ShardedBloomCounter(a.size, a.fpr, k=a.mer_len, canonical=a.canonical, rank=rank, world=world, device=local)
    if a.split == "files":
        add_files(sbc, a.files, rank, world)
    elif not add_split(sbc, a.files, rank, world, a.mer_len):
        if rank == 0:
            sys.stderr.write("bc_multi: a FASTQ share does not start on a record; counting whole files per rank instead\n")
        sbc.bc.hc.clear()
        add_files(sbc, a.files, rank, world)
    sbc.dump_slice(a.output)
    if world > 1:
        dist.barrier()
    if rank == 0:
        cmdline = ["bc_multi"] + (argv if argv is not None else sys.argv[1:])
        concat_bloom_slices(a.output, world, sbc.header(cmdline), a.output)
        if not a.keep_shards:
            for r in range(world):
                os.unlink("%s.%d" % (a.output, r))
        sys.stderr.write("bc_multi: %d GPUs, output %s\n" % (world, a.output))
    sbc.close()
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
