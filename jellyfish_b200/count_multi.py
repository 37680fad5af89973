"""`jellyfish count` over several GPUs of one node.

    torchrun --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 -m jellyfish_b200.count_multi \
        -m 21 -s 16G -C -o mer_counts.jf reads_1.fa reads_2.fa ...

With `--split auto` (the default) every file is split among the ranks (jellyfish_b200/split.py): rank r counts the bytes
from the first line start at or after r/N of the file -- for FASTQ the first line where two records look whole -- up to
where rank r+1's share starts.  A FASTA share that starts in the middle of a sequence first parses a seam of whole lines in
front of it without counting them (jfgpu_seam), so the k-mers that span the cut are counted once, by the rank the cut
starts.  Each rank reads its share with pread into two pinned buffers of one exchange round each, so a file may be larger
than host or device memory.  The FASTQ cuts are checked after the count: every rank tallies the newlines of its share on
the device and the tallies are gathered; if a share does not start behind a multiple of 4 lines (a sequence line that
starts with '@' and a quality line that starts with '+' can fool the local rule), every rank clears its table and the
files are counted again with `--split files`, with a note on stderr.  A path that is not a regular file (a pipe, a
process substitution such as `<(zcat reads.fq.gz)`) cannot be read at offsets: it is counted whole by one rank, as with
`--split files`.  `--split files`: every rank parses the files
`files[rank::N]` whole (a file is the unit of distribution: no k-mer spans two
files, mer_overlap_sequence_parser.hpp:111).  Either way the k-mers are routed to the rank that owns their table
position, each rank writes `OUT.<rank>`, and rank 0 concatenates the shards in rank order into OUT --
byte-identical to what one GPU (or the reference) writes for the same input, since shard r holds
exactly the positions r*size/N ... (r+1)*size/N - 1.  (`jellyfish merge` on the shard files gives the
same records: jellyfish/merge_files.cc:45-176.)  -m takes 1..128; k > 64 (32-byte keys) is routed by the key exchange
on 2, 4 or 8 GPUs, with 64 MB batches.

`--sam PATH` (may be given several times; read after the positional files) counts the reads of SAM text, gzip'd SAM and
BAM files, each record's SEQ with its QUAL as one FASTQ read, as the single-GPU `count --sam` does
(jellyfish_b200/split_sam.py).  With `--split auto`, SAM text is cut at line starts and BAM at a BGZF block and the first
record behind it; every rank inflates its own blocks on a pool of threads.  Each piece is turned into FASTQ on the device
(jfgpu_sam_stage) and routed as FASTQ.  A BAM rank's records must end exactly where the next rank's start: when they do
not, every rank clears its table and counts whole files, with a note on stderr.  gzip'd SAM and pipes are counted whole by
one rank; CRAM is refused.

`-Q CHAR` (or `--min-quality N` with `--quality-start Q`) leaves out the bases whose quality character is below the
threshold, as the single-GPU `count -Q` does.  A feed of FASTQ text must then end behind a whole record, so the text is cut
there: a whole file in device memory into exchange rounds by one device pass (jfgpu_fastq_cuts), a share into pieces on
the reading thread.  A FASTA file is split at header lines only (no seam is parsed), so a file of fewer records than
ranks leaves some ranks idle.  `--if FILE` (may be given several times) counts only the k-mers of those files: every rank
primes their k-mers (split among the ranks like any input, with neither the quality filter nor a Bloom structure), drains,
and only then every rank counts the inputs into the primed keys.  When a cut check fails, both passes are repeated with
whole files.  A FASTQ record longer than a quarter of a piece, or (for a file counted whole) than an exchange round, is an
error of the rank that reads it: with two or more ranks the others then wait for it until the launcher's timeout.

Bloom structures (k <= 64) take the key exchange: `--bc FILE` is loaded whole by every rank and tested before a k-mer is
routed; `--bf-size N` (the GLOBAL expected number of k-mers) gives every rank a filter for its share, applied by the
owner after the exchange, where every occurrence of a k-mer arrives.

`--disk`: a shard never doubles; when this rank's shard is full it is written to `OUT.<rank>.<i>` (i = 0, 1, ...), zeroed,
and counting goes on, with no wait for the other ranks.  At the end a rank that never spilled writes `OUT.<rank>` with
-L/-U as usual; a rank that spilled writes its table as one more piece, merges its pieces into `OUT.<rank>` (the `merge`
of the command-line driver, -L/-U applied to the sums) and deletes them unless `--no-unlink` is given; rank 0
concatenates.  The result is the single-GPU `count --disk` output for any world size.  `--no-merge` (once some rank has
spilled) leaves every rank's pieces and writes no OUT: `jellyfish merge -o OUT OUT.*.*` gives it.  When a cut check fails
every rank deletes its pieces before the files are counted again.  `--disk --if` is refused.  Without `--disk`,
`--no-merge` and `--no-unlink` do nothing.
"""
import argparse
import datetime
import os
import sys
import time

import torch
import torch.distributed as dist

from . import split_sam
from .engine import HashCounter, JellyfishError
from .distributed import ShardedCounter, ShareReader, all_ranks_ok, concat_shards, fastq_cuts_agree
from .split import plan_file, splittable


def _size(v):
    mult = {"k": 10**3, "M": 10**6, "G": 10**9, "T": 10**12}
    return int(v[:-1]) * mult[v[-1]] if v[-1] in mult else int(v)


# An error found by one rank alone (a FASTQ record too long for a piece or a round under -Q, a run of '\r' where a share is
# cut) ends that rank; the others are then left in the next collective until the job launcher's timeout ends them.
_PEERS_WAIT = " (this rank stops here; the other ranks wait for it until the launcher's timeout)"

# --disk: how long a rank waits in a collective for the others (NCCL's default is 10 minutes), long enough for a peer that
# writes a full shard or merges its pieces on the CPU
DISK_TIMEOUT_S = 6 * 3600


def _count_whole(sc, path, owner):
    """One file read whole by one rank and counted from device memory; every other rank takes part in the exchange rounds."""
    if not owner:
        sc.add_device_text(0, 0)
        return
    with open(path, "rb") as f:
        data = f.read()
    if data[:1] not in (b">", b"@", b""):
        raise SystemExit("Unsupported format: %s" % path)
    buf = torch.zeros(max(16, len(data) + 256), dtype=torch.uint8, device="cuda")
    if data:
        buf[:len(data)] = torch.frombuffer(bytearray(data), dtype=torch.uint8).cuda()
    sc.add_device_text(buf.data_ptr(), len(data), fastq=data[:1] == b"@")


def count_files(sc, files, rank, world):
    """--split files: rank r counts files[r::world], each whole and resident in device memory."""
    mine = files[rank::world]
    rounds = torch.tensor([len(mine)], device="cuda")
    if world > 1:
        dist.all_reduce(rounds, op=dist.ReduceOp.MAX)       # every rank takes part in every exchange
    for i in range(int(rounds.item())):
        if i < len(mine):
            _count_whole(sc, mine[i], True)
        else:
            sc.add_device_text(0, 0)


def count_split(sc, files, rank, world, k):
    """--split auto: every regular file split among the ranks and streamed (see the module documentation); anything else
    (a pipe, a process substitution) counted whole by rank i % world, as --split files would.  Returns False when a FASTQ
    share did not start on a record: the table then holds a wrong count and must be cleared."""
    tallies = []
    for i, path in enumerate(files):
        if not splittable(path):
            _count_whole(sc, path, i % world == rank)
            continue
        try:
            share = plan_file(path, rank, world, k, headers=sc.qual)
        except ValueError:
            raise SystemExit("Unsupported format: %s" % path)
        if share is None:                      # an empty file holds no k-mer
            continue
        reader = ShareReader(path, share, sc.piece_bytes(), records=sc.qual and share.fmt == "fastq")
        try:
            seam = reader.seam()
            if seam:
                t = torch.frombuffer(bytearray(seam), dtype=torch.uint8).cuda()
                sc.hc.seam(t.data_ptr(), len(seam), fmt=share.fmt)
                del t
            tally = torch.zeros(1, dtype=torch.int64, device="cuda") if share.fmt == "fastq" else None
            sc.add_pieces(reader, tally)
        except ValueError as ex:               # (a record too long for a piece)
            raise SystemExit("%s: %s%s" % (path, ex, _PEERS_WAIT if world > 1 else ""))
        finally:
            reader.close()
        if tally is not None:
            tallies.append([share.end - share.start, int(tally.item())])
    return fastq_cuts_agree(tallies, world, "cuda")


def _count_sam_reader(sc, path, reader, tolerant=False):
    """A corrupt or truncated BGZF block (found while inflating, on the reader's thread) is a one-line error."""
    try:
        return sc.add_sam_pieces(reader, tolerant)
    except ValueError as ex:
        raise SystemExit("%s: %s" % (path, ex))
    finally:
        reader.close()
        sc.sam_inflate_s += getattr(reader, "inflate_s", 0.0)


def _whole_sam(sc, path, owner):
    try:
        reader = split_sam.whole_reader(path, owner, sc.sam_piece_bytes())
    except ValueError as ex:
        raise SystemExit("%s: %s" % (path, ex))
    _count_sam_reader(sc, path, reader)


def count_sam_files(sc, sams, rank, world):
    """--split files (and the fall-back): rank r counts the SAM / BAM files sams[r::world] whole."""
    t0 = time.perf_counter()
    for i, path in enumerate(sams):
        _whole_sam(sc, path, i % world == rank)
    sc.sam_wall_s += time.perf_counter() - t0


def count_sam_split(sc, sams, rank, world):
    """--split auto for --sam files: SAM text and BAM split among the ranks, anything else counted whole by rank i % world.
    Returns False on this rank when one of its shares could not be counted on its own (a BAM record chain that does not end
    where the next share starts): the table then holds a wrong count and must be cleared."""
    ok = True
    t0 = time.perf_counter()
    for i, path in enumerate(sams):
        k = split_sam.kind(path) if splittable(path) else "pipe"
        if k == "cram":
            raise SystemExit("CRAM input is not supported ('%s')" % path)
        if k not in ("sam", "bam"):
            if k is not None:
                _whole_sam(sc, path, i % world == rank)
            continue
        try:
            kind_, share = split_sam.plan_file(path, rank, world, k)
            if kind_ == "sam":
                reader = split_sam.SamShareReader(path, share, sc.sam_piece_bytes())
            else:
                reader = split_sam.BamShareReader(path, share, sc.sam_piece_bytes())
        except ValueError as ex:
            raise SystemExit("%s: %s" % (path, ex))
        ok = _count_sam_reader(sc, path, reader, tolerant=True) and ok
    sc.sam_wall_s += time.perf_counter() - t0
    return ok


def parse_args(argv=None):
    """The command line, checked as the single-GPU command checks it (exits on an error)."""
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
    ap.add_argument("--split", choices=("auto", "files"), default="auto",
                    help="auto: split every file among the ranks; files: give rank r the whole files files[r::N]")
    ap.add_argument("--sam", action="append", default=[], metavar="PATH",
                    help="SAM, gzip'd SAM or BAM file to count (may be given several times)")
    ap.add_argument("-Q", "--min-qual-char", help="bases whose quality character is below this one are not counted")
    ap.add_argument("--min-quality", type=int, help="-Q as a number: the quality character --quality-start + N")
    ap.add_argument("--quality-start", type=int, default=64, help="the quality character of --min-quality 0")
    ap.add_argument("--if", dest="if_files", action="append", default=[], metavar="PATH",
                    help="count only the k-mers of this file (may be given several times)")
    ap.add_argument("--disk", action="store_true",
                    help="a full shard is written to OUT.<rank>.<i>, zeroed, and counting goes on; the pieces are merged at the end")
    ap.add_argument("--no-merge", action="store_true", help="--disk: leave the pieces OUT.<rank>.<i> and write no OUT")
    ap.add_argument("--no-unlink", action="store_true", help="--disk: keep the pieces after merging them")
    ap.add_argument("files", nargs="*")
    a = ap.parse_args(argv)

    def error(msg):
        sys.stderr.write("Error: %s\n" % msg)
        sys.exit(1)
    # the single-GPU command's checks (count_main.cc:196-197,234-256 and the k <= 64 scope of every Bloom structure)
    if a.bf_size and a.bc:
        error("Switches [--bf-size] and [--bc] conflict")
    a.min_qual = 0
    if a.min_qual_char is not None:
        if len(a.min_qual_char.encode()) != 1:
            error("[-Q, --min-qual-char] must be one character.")
        if not "!" <= a.min_qual_char <= "~":
            error("Quality character '%s' is outside of the range [!, ~]" % a.min_qual_char)
        a.min_qual = ord(a.min_qual_char)
    if a.min_quality is not None:
        if not 33 <= a.quality_start <= 126:
            error("Quality start %d is outside the range [33, 126]" % a.quality_start)
        mq = a.quality_start + a.min_quality
        if not 33 <= mq <= 126:
            error("Min quality %d is outside the range [0, %d]" % (a.min_quality, 126 - a.quality_start))
        a.min_qual = mq
    if not a.files and not a.sam:
        ap.error("no input file: give sequence files or --sam")
    if a.mer_len > 64 and (a.bf_size or a.bc):
        sys.stderr.write("Error: --bf-size and --bc take mer lengths up to 64\n")
        sys.exit(1)
    if a.disk and a.if_files:
        # which primed keys a spill keeps depends on when each shard fills: no count of the reference's to be held to
        error("--disk with --if is not supported on several GPUs (the keys primed before a spill would be lost)")
    return a


def main(argv=None):
    a = parse_args(argv)
    rank, world = int(os.environ.get("RANK", "0")), int(os.environ.get("WORLD_SIZE", "1"))
    local = int(os.environ.get("LOCAL_RANK", rank))
    torch.cuda.set_device(local)
    if world > 1:
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        os.environ.setdefault("NCCL_MAX_CTAS", "16")      # K1 leaves 16 SMs to the exchange that runs beside it
        # --disk: a rank that spills or merges keeps the others waiting in the next collective or the final barrier
        timeout = {"timeout": datetime.timedelta(seconds=DISK_TIMEOUT_S)} if a.disk else {}
        dist.init_process_group("nccl", device_id=torch.device("cuda", local), **timeout)
    run(a, argv, rank, world, local)


def run(a, argv, rank, world, local):
    """Count and write the output on this rank of an initialised process group (world 1: none); an engine error is a
    one-line message and exit status 1."""
    try:
        _count(a, argv, rank, world, local)
    except JellyfishError as ex:
        sys.stderr.write("count_multi: %s%s\n" % (ex, _PEERS_WAIT if world > 1 else ""))
        sys.exit(1)


def _prime(sc, a, count):
    """--if (count_main.cc:288-295): every rank primes the k-mers of the --if files with count(files), then switches to
    UPDATE for the inputs.  Returns what count returns (True without --if)."""
    if not a.if_files:
        return True
    sc.set_op(HashCounter.OP_PRIME)
    ok = count(a.if_files)
    sc.set_op(HashCounter.OP_UPDATE)
    return ok is not False


def _count(a, argv, rank, world, local):
    sc = ShardedCounter(a.size, a.counter_len, k=a.mer_len, canonical=a.canonical, rank=rank, world=world, device=local,
                        reprobes=a.reprobes, bf_size=a.bf_size, bf_fp=a.bf_fp, bc=a.bc, min_qual=a.min_qual,
                        disk=a.output if a.disk else None, out_counter_len=a.out_counter_len)
    sc.sam_inflate_s = sc.sam_wall_s = 0.0
    if a.split == "files":
        _prime(sc, a, lambda files: count_files(sc, files, rank, world))
        count_files(sc, a.files, rank, world)
        count_sam_files(sc, a.sam, rank, world)
    else:
        prime_ok = _prime(sc, a, lambda files: count_split(sc, files, rank, world, a.mer_len))
        fastq_ok = count_split(sc, a.files, rank, world, a.mer_len) and prime_ok
        sam_ok = all_ranks_ok(count_sam_split(sc, a.sam, rank, world), world, "cuda")
        if not (fastq_ok and sam_ok):
            if rank == 0:
                what = "a FASTQ share does not start on a record" if not fastq_ok else \
                    "a SAM/BAM share could not be counted on its own (a BAM record chain does not meet the next share)"
                sys.stderr.write("count_multi: %s; counting whole files per rank instead\n" % what)
            if sc.disk:
                sc.disk.discard_pieces()     # (no piece of the abandoned pass may reach the merge)
            sc.hc.clear()
            _prime(sc, a, lambda files: count_files(sc, files, rank, world))
            count_files(sc, a.files, rank, world)
            count_sam_files(sc, a.sam, rank, world)
    st = sc.done()
    if a.sam:
        # (read by scripts/sam_multi_bench.py)
        sys.stderr.write("count_multi: rank %d --sam times: inflate_s %.4f transcode_route_s %.4f sam_wall_s %.4f\n"
                         % (rank, sc.sam_inflate_s, sc.sam_device_s, sc.sam_wall_s))
    cmdline = ["count_multi"] + (argv if argv is not None else sys.argv[1:])
    shard = "%s.%d" % (a.output, rank)
    if not a.disk:
        sc.hc.dump(shard, lower=a.lower_count, upper=a.upper_count, out_counter_len=a.out_counter_len, cmdline=cmdline)
        pieces_only = False
    else:
        # --no-merge leaves pieces only once some rank has spilled: a count that never filled a shard writes OUT, as the
        # single-GPU count --disk does
        pieces_only = a.no_merge and not all_ranks_ok(not sc.disk.pieces, world, "cuda")
        spills = len(sc.disk.pieces)
        merge_s = sc.disk.write_output(shard, a.lower_count, a.upper_count, cmdline, merge=not pieces_only, unlink=not a.no_unlink)
        # (read by scripts/disk_multi_bench.py)
        sys.stderr.write("count_multi: rank %d --disk: spills %d spill_s %.4f merge_s %.4f\n" % (rank, spills, sc.disk.spill_s, merge_s))
    if world > 1:
        dist.barrier()
    if pieces_only:
        if rank == 0:
            sys.stderr.write("count_multi: --no-merge: pieces %s.<rank>.<i> left for `jellyfish merge`\n" % a.output)
    elif rank == 0:
        concat_shards(a.output, world, a.output)
        if not a.keep_shards:
            for r in range(world):
                os.unlink("%s.%d" % (a.output, r))
        sys.stderr.write("count_multi: %d GPUs, %d k-mers on rank 0's share, output %s\n" % (world, st["kmers"], a.output))
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
