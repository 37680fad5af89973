"""Time `count_multi --sam` on one large BAM, and on the same reads as SAM text, at N = 1, 2, 4 and 8 GPUs (those present).

    python scripts/sam_multi_bench.py [--worlds 1,2,4,8] [--reads 5000000] [--k 21] [--dir DIR] [--out FILE]

The input is `--reads` reads of 150 bases (iid ACGT and qualities from a seeded numpy generator) written as SAM text with
realistic fields, and as BAM in BGZF blocks of 64 KB of inflated data (zlib level 6, as samtools writes).  Every file is
read once before it is timed (a warm page cache: this script changes no system setting).  For each world N and form,
`count_multi -m K -s SIZE -C --sam FILE` runs once (plain python for N = 1, torchrun above), and for the BAM also with
`--split files` (the file read whole by one rank, block by block).  Every rank reports:

  inflate_s          wall time of reading and inflating its BGZF blocks (on the prefetch thread, beside the device work);
  transcode_route_s  host time of transcoding its pieces (jfgpu_sam_stage) and routing their FASTQ (the extraction into
                     the exchange buffers), both synchronised; with one rank, of transcoding and counting them;
  sam_wall_s         wall time of its whole --sam phase: inflating, transcoding, routing and the exchange rounds.

and the command's wall time (process start, NCCL set-up, table allocation and the dump included).  The single-GPU
`jellyfish-b200 count --sam` of each file is timed too (wall time of the command), as the yardstick.  The GPU's name, power
limit and SM clocks are read in the same run.  Prints one JSON line; --out also writes it to a file.
"""
import argparse
import json
import os
import re
import struct
import subprocess
import sys
import tempfile
import time
import zlib

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
READ = 150
BLOCK = 65280


def write_inputs(sam_path, bam_path, n_reads, seed):
    """The same reads as SAM text and as BGZF-compressed BAM (refID -1: unmapped, CIGAR '*')."""
    rng = np.random.default_rng(seed)
    lut = np.frombuffer(b"ACGT", np.uint8)
    codes = np.frombuffer(b"\x01\x02\x04\x08", np.uint8)
    header = b"@HD\tVN:1.6\tSO:unsorted\n"
    bam_head = b"BAM\1" + struct.pack("<i", len(header)) + header + struct.pack("<i", 0)
    pending = bytearray(bam_head)
    with open(sam_path, "wb") as fs, open(bam_path, "wb") as fb:
        fs.write(header)
        step = 100000
        for q in range(0, n_reads, step):
            m = min(step, n_reads - q)
            b = rng.integers(0, 4, (m, READ), dtype=np.uint8)
            qual = rng.integers(2, 41, (m, READ), dtype=np.uint8)
            seqs, quals = lut[b], qual + 33
            packed = (codes[b[:, 0::2]] << 4) | codes[b[:, 1::2]]
            lines = []
            for i in range(m):
                name = b"r%d" % (q + i)
                lines.append(b"%s\t4\t*\t0\t0\t*\t*\t0\t0\t%s\t%s\n" % (name, seqs[i].tobytes(), quals[i].tobytes()))
                body = struct.pack("<iiBBHHHiiii", -1, -1, len(name) + 1, 0, 4680, 0, 4, READ, -1, -1, 0)
                body += name + b"\0" + packed[i].tobytes() + qual[i].tobytes()
                pending += struct.pack("<I", len(body)) + body
            fs.write(b"".join(lines))
            while len(pending) >= BLOCK:
                fb.write(_bgzf_block(bytes(pending[:BLOCK])))
                del pending[:BLOCK]
        if pending:
            fb.write(_bgzf_block(bytes(pending)))
        fb.write(_bgzf_block(b""))


def _bgzf_block(data):
    c = zlib.compressobj(6, zlib.DEFLATED, -15)
    cdata = c.compress(data) + c.flush()
    head = b"\x1f\x8b\x08\x04\x00\x00\x00\x00\x00\xff" + struct.pack("<HBBHH", 6, ord("B"), ord("C"), 2, 18 + len(cdata) + 8 - 1)
    return head + cdata + struct.pack("<II", zlib.crc32(data), len(data))


def warm(path):
    with open(path, "rb") as f:
        while f.read(64 << 20):
            pass


TIMES = re.compile(r"rank (\d+) --sam times: inflate_s ([\d.]+) transcode_route_s ([\d.]+) sam_wall_s ([\d.]+)")


def run(world, args, port):
    env = dict(os.environ, SOURCE_DATE_EPOCH="0")
    cmd = [sys.executable, "-m"] if world == 1 else [sys.executable, "-m", "torch.distributed.run", "--nnodes=1",
                                                     "--nproc-per-node", str(world), "--master-addr", "127.0.0.1",
                                                     "--master-port", str(port), "-m"]
    t0 = time.perf_counter()
    r = subprocess.run(cmd + ["jellyfish_b200.count_multi"] + args, cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
    dt = time.perf_counter() - t0
    out = r.stdout.decode(errors="replace")
    if r.returncode:
        raise SystemExit(out[-3000:])
    ranks = sorted((int(m[0]), float(m[1]), float(m[2]), float(m[3])) for m in TIMES.findall(out))
    return dt, [{"rank": r_, "inflate_s": a, "transcode_route_s": b, "sam_wall_s": c} for r_, a, b, c in ranks]


def run_one_gpu(args):
    """wall time of the single-GPU command-line `count` with these arguments"""
    env = dict(os.environ, SOURCE_DATE_EPOCH="0")
    t0 = time.perf_counter()
    r = subprocess.run([os.path.join(ROOT, "jellyfish_b200", "lib", "jellyfish-b200"), "count"] + args, cwd=ROOT, env=env,
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
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
    ap.add_argument("--reads", type=int, default=5000000)
    ap.add_argument("--k", type=int, default=21)
    ap.add_argument("--dir", default=None, help="local disk for the inputs (default: a temporary directory)")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    n_dev = torch.cuda.device_count()
    if n_dev == 0:
        raise SystemExit("sam_multi_bench: no CUDA device")
    worlds = [w for w in (int(x) for x in a.worlds.split(",")) if w <= n_dev]
    res = {"bench": "sam_multi", "k": a.k, "reads": a.reads, "read_len": READ, "gpu": gpu_info(), "page_cache": "warm", "runs": []}
    size = 1 << max(20, int(np.ceil(np.log2(a.reads * READ * 1.25))))
    with tempfile.TemporaryDirectory(dir=a.dir) as d:
        sam, bam = os.path.join(d, "reads.sam"), os.path.join(d, "reads.bam")
        write_inputs(sam, bam, a.reads, seed=7)
        res["bytes"] = {"sam": os.path.getsize(sam), "bam": os.path.getsize(bam)}
        out = os.path.join(d, "out.jf")
        base = ["-m", str(a.k), "-s", str(size), "-C", "-o", out]
        for form, path in (("bam", bam), ("sam", sam)):
            warm(path)
            res["runs"].append({"command": "count", "form": form, "wall_s": round(run_one_gpu(base + ["--sam", path]), 3)})
            os.unlink(out)
        for world in worlds:
            for form, path, split in (("bam", bam, "auto"), ("bam", bam, "files"), ("sam", sam, "auto")):
                warm(path)
                dt, ranks = run(world, base + ["--split", split, "--sam", path], 29800 + world)
                res["runs"].append({"command": "count_multi", "world": world, "form": form, "split": split, "wall_s": round(dt, 3),
                                    "ranks": ranks})
                os.unlink(out)
    res["gpu_after"] = gpu_info()
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
