"""One process per GPU: the hash table sharded by the top bits of the hash position.

The reference is a single process (SURVEY.md section 2a); this module is the multi-GPU form of
`hash_counter`: every rank parses its own part of the input, the canonical k-mers are bucketed
by the rank that owns their table position (device kernel, `jfgpu_extract_route`), exchanged
with one NCCL all-to-all per batch, and inserted by their owner (`jfgpu_insert_keys`).  All
ranks draw the same hash matrix (the reference's deterministic random stream), and shard r owns
the positions whose top log2(world) bits equal r, so the rank-ordered concatenation of the
shard dumps is byte-identical to the single-GPU dump.

Two forms of the exchange: 4-byte region RECORDS (RecordExchange, the default where the table geometry allows it: k <= 21,
32-bit slots) and packed KEYS (any geometry: 8, 16 or 32 bytes a key for k <= 32, k <= 64 and k <= 128).  The exchange logic (bucket capacities, count exchange, uneven all-to-all,
ordering of the shard files) is plain torch.distributed code and is exercised on CPU with the gloo backend in
tests/test_distributed_cpu.py through the `RouteBackend` seam below.
"""
import os
import time

import torch
import torch.distributed as dist

UINT64_MAX = (1 << 64) - 1


class RouteBackend(object):
    """What the exchange needs from the engine; the CUDA engine implements it with kernels."""

    key_words = 1

    def extract_route(self, text, begin, end, keys, capacity, counts):
        raise NotImplementedError

    def insert_keys(self, keys, n):
        raise NotImplementedError


class EngineBackend(RouteBackend):
    """libjfgpu.so (sm_90a kernels) behind the seam."""

    def __init__(self, hc):
        self.hc = hc
        self.key_words = hc.key_words

    def extract_route(self, text, begin, end, keys, capacity, counts):
        # the engine works on torch's current stream, so its kernels are ordered with the NCCL
        # collectives and the tensor ops around them
        ptr, n = text
        self.hc.extract_route(ptr, n, keys.data_ptr(), capacity, counts.data_ptr(), begin=begin, end=end,
                              stream=torch.cuda.current_stream().cuda_stream)

    def insert_keys(self, keys, n):
        if n:
            self.hc.insert_keys(keys.data_ptr(), n, stream=torch.cuda.current_stream().cuda_stream)


def exchange_and_insert(backend, world, send, counts, capacity, recv, before_payload=None):
    """Uneven all-to-all of the bucketed keys, then insertion on the owner.

    send:   int64 tensor [world, capacity * key_words]; bucket d holds counts[d] keys for rank d
    counts: int64 tensor [world] (device of `send`)
    recv:   int64 tensor [world, capacity * key_words] scratch
    before_payload: optional callable run after the (host-synchronising) count exchange and before
        the payload exchange -- the pipelined caller launches the next batch's extraction there, so
        that it overlaps the NVLink transfer and the insertion of this batch.
    Returns the number of keys this rank received."""
    kw = backend.key_words
    if world == 1:
        n = int(counts[0].item())
        if before_payload:
            before_payload()
        backend.insert_keys(send[0], n)
        return n
    recv_counts = torch.empty_like(counts)
    dist.all_to_all_single(recv_counts, counts)
    sc = counts.tolist()
    rc = recv_counts.tolist()
    if max(sc) > capacity or max(rc) > capacity:
        raise RuntimeError("route bucket capacity exceeded (%d > %d)" % (max(max(sc), max(rc)), capacity))
    if before_payload:
        before_payload()
    total = sum(rc)
    flat_out = recv.view(-1)[:total * kw]
    if dist.get_backend() == "nccl":
        # list form: the buckets are sent straight from where the kernel wrote them (no packing copy)
        outs, o = [], 0
        for s in range(world):
            outs.append(flat_out[o:o + rc[s] * kw])
            o += rc[s] * kw
        dist.all_to_all(outs, [send[d, :sc[d] * kw] for d in range(world)])
    else:
        flat_in = torch.cat([send[d, :sc[d] * kw] for d in range(world)])
        dist.all_to_all_single(flat_out, flat_in, output_split_sizes=[c * kw for c in rc], input_split_sizes=[c * kw for c in sc])
    backend.insert_keys(flat_out, total)
    return total


CHUNK = 8192          # bytes of a record chunk (jf_kernels.cuh CHUNK_BYTES)


class _DeviceBytes(object):
    """A byte range of device memory, seen by torch (CUDA array interface)."""

    def __init__(self, ptr, n):
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": "|u1", "data": (ptr, False), "version": 2}


def aligned_text(ptr, n, stage):
    """ptr when it is 16-byte aligned (what the extraction takes), else the n bytes copied to the device tensor `stage` on
    torch's current stream: a round of device text cut behind a FASTQ record starts anywhere."""
    if ptr % 16 == 0 or n == 0:
        return ptr
    stage[:n].copy_(torch.as_tensor(_DeviceBytes(ptr, n), device=stage.device))
    return stage.data_ptr()


class RecordExchange(object):
    """The record form of the exchange (include/jfgpu.h, jfgpu_shard_*): every rank's K1 writes 4-byte records of the GLOBAL
    table's regions into a send pool whose chunk arenas belong to the owning shards; the chunks cross NVLink as they are
    (one NCCL all-to-all per round, list form: no packing copy), the owner re-files them under its own regions
    (restage_kernel) and drains them like a single GPU.  Two send banks: the extraction of round r+1 (stream A) runs beside
    the exchange and the restaging of round r (stream B)."""

    def __init__(self, hc, world, rank, dev, send_gb=None):
        self.hc, self.world, self.rank, self.dev = hc, world, rank, dev
        self.ok = False
        self.trace = None
        if not hc.shard_setup(0, 0, 0, 0, 0, 0):       # geometry probe: nothing is allocated for tables the record form does not cover
            return
        free, _ = torch.cuda.mem_get_info(dev)
        # two send banks + one receive pool = 3 x world x arena; a quarter of the free memory, at most 36 GB, for the three
        budget = min(free // 4, 36 << 30) if send_gb is None else int(send_gb * (1 << 30))
        n_sm = torch.cuda.get_device_properties(dev).multi_processor_count
        floor = 2 * n_sm * max(1, 1024 // world) + 64
        self.arena = max(floor, budget // (3 * world * (CHUNK + 8)))
        try:
            self.send = torch.empty(2 * world * self.arena * CHUNK, dtype=torch.uint8, device=dev)
            self.send_dir = torch.empty(2 * world * self.arena * 8, dtype=torch.uint8, device=dev)
            self.recv = torch.empty(world * self.arena * CHUNK, dtype=torch.uint8, device=dev)
            self.recv_dir = torch.empty(world * self.arena * 8, dtype=torch.uint8, device=dev)
        except RuntimeError:
            return
        if not hc.shard_setup(self.send.data_ptr(), self.send_dir.data_ptr(), self.arena, self.recv.data_ptr(), self.recv_dir.data_ptr(), self.arena):
            self.send = self.send_dir = self.recv = self.recv_dir = None
            return
        self.round_bytes = hc.shard_round_bytes()
        if self.round_bytes < (1 << 20):
            return
        # the chunk counts travel on a communicator of their own, so that they never queue behind the chunks of the round before
        self.pg_counts = dist.new_group(backend="nccl") if dist.get_backend() == "nccl" else None
        self.sa = torch.cuda.Stream(device=dev)       # extraction
        self.sb = torch.cuda.Stream(device=dev)       # exchange + restaging
        self.sent = [torch.cuda.Event(), torch.cuda.Event()]     # bank b has been sent (may be overwritten)
        self.ok = True

    def _views(self, pool, bank, counts, unit):
        w, a = self.world, self.arena
        return [pool[((bank * w + d) * a) * unit:((bank * w + d) * a + counts[d]) * unit] for d in range(w)]

    def add_device_text(self, ptr, n, begin, end, bounds=None):
        """bounds: the piece bounds of the rounds ([0, ..., n], record_bounds); None: rounds of round_bytes."""
        self._rounds(n, begin, end, lambda off, ln, bank: aligned_text(ptr + off, ln, self._stage_buf(bank)), bounds)

    def _stage_buf(self, bank):
        if getattr(self, "_stage", None) is None:
            self._stage = [torch.empty(self.round_bytes + 256, dtype=torch.uint8, device=self.dev) for _ in range(2)]
        return self._stage[bank]

    def _staged(self, hptr, ln, bank):
        """Copy ln bytes of pinned host text into the device staging buffer of `bank` on the extraction stream."""
        import ctypes as C
        from . import _lib
        dst = self._stage_buf(bank).data_ptr()
        if ln and _lib.load().jfgpu_memcpy_h2d(C.c_void_p(dst), C.c_void_p(hptr), ln, C.c_void_p(self.sa.cuda_stream)):
            raise RuntimeError("host to device copy failed")
        return dst

    def add_host_text(self, hptr, n, begin, end):
        """Pinned host text: every round's slice is copied to a device staging buffer (one per bank) on the extraction stream."""
        self._rounds(n, begin, end, lambda off, ln, bank: self._staged(hptr + off, ln, bank))

    def add_pieces(self, reader, tally=None):
        """A share of a file, piece by piece (ShareReader): piece i is read into pinned memory, copied to the staging buffer
        of its bank and extracted while the exchange of piece i - 1 runs.  tally: a device int64 the newlines of every piece
        are added to."""
        def extract(r, bank):
            if r >= reader.n_pieces:
                return
            hptr, ln, begin, end = reader.read(r)
            src = self._staged(hptr, ln, bank)
            reader.release(r, self.sa)
            reader.prefetch(r + 1)
            if tally is not None:
                self.hc.count_newlines(src, ln, tally.data_ptr(), stream=self.sa.cuda_stream)
            self.hc.shard_extract(src, ln, bank, begin, end, stream=self.sa.cuda_stream, fmt=reader.fmt)
        self._run(reader.n_pieces, extract)

    def add_sam_pieces(self, n_pieces, stage):
        """SAM / BAM pieces: stage(i, stream) transcodes piece i into FASTQ of whole records in device memory -> (pointer,
        bytes), which round i extracts as a FASTQ file of its own.  Both run on the host thread while stream B exchanges
        and restages round i - 1.  Returns the host time of the stages and extractions (both synchronise)."""
        spent = [0.0]

        def extract(r, bank):
            t0 = time.perf_counter()
            ptr, n = stage(r, self.sa)
            if n:
                self.hc.shard_extract(ptr, n, bank, True, True, stream=self.sa.cuda_stream, fmt="fastq")
            spent[0] += time.perf_counter() - t0
        self._run(n_pieces, extract)
        return spent[0]

    def _rounds(self, n, begin, end, fetch, bounds=None):
        if bounds is None:
            bounds = [min(n, r * self.round_bytes) for r in range((n + self.round_bytes - 1) // self.round_bytes + 1)] if n else [0]
        rounds = len(bounds) - 1

        def extract(r, bank):
            off = bounds[r] if r < rounds else n
            ln = bounds[r + 1] - off if r < rounds else 0
            if ln or (r == 0 and begin) or (r == rounds_all[0] - 1 and end):
                src = fetch(off, ln, bank)
                self.hc.shard_extract(src, ln, bank, begin and r == 0, end and off + ln >= n, stream=self.sa.cuda_stream)
        rounds_all = [0]
        self._run(rounds, extract, rounds_all)

    def _run(self, rounds, extract, rounds_out=None):
        """Every rank takes part in max(rounds over the ranks, 1) exchange rounds; extract(r, bank) files round r's records
        into send bank `bank` on the extraction stream (nothing when this rank has no text for the round)."""
        w = self.world
        t = torch.tensor([rounds], dtype=torch.int64, device=self.dev)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        rounds_all = max(int(t.item()), 1)        # every rank takes part in every exchange
        if rounds_out is not None:
            rounds_out[0] = rounds_all
        for ev in self.sent:
            ev.record(self.sb)
        marks = []                                  # CUDA events around the stages of every round (self.trace)
        for r in range(rounds_all):
            bank = r & 1
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(5)]
            marks.append(ev)
            with torch.cuda.stream(self.sa):
                self.sa.wait_event(self.sent[bank])
                ev[0].record(self.sa)
                extract(r, bank)
                ev[1].record(self.sa)
                counts = self.hc.shard_pack(bank, stream=self.sa.cuda_stream)       # synchronises stream A
                sc = torch.tensor(counts, dtype=torch.int64, device=self.dev)
                rc = torch.empty_like(sc)
                dist.all_to_all_single(rc, sc, group=self.pg_counts)
                rcl = rc.tolist()                  # (waits for this tiny exchange only: stream B keeps working on the round before)
                if max(rcl) > self.arena:
                    raise RuntimeError("route bucket capacity exceeded (%d chunks > %d)" % (max(rcl), self.arena))
            with torch.cuda.stream(self.sb):
                ev[2].record(self.sb)
                # this rank's own chunks do not travel: the restaging reads them where K1 left them
                me = self.rank
                outs = [self.recv[(s * self.arena) * CHUNK:(s * self.arena + (0 if s == me else rcl[s])) * CHUNK] for s in range(w)]
                ins = self._views(self.send, bank, [0 if d == me else c for d, c in enumerate(counts)], CHUNK)
                dist.all_to_all(outs, ins)
                outs_d = [self.recv_dir[(s * self.arena) * 8:(s * self.arena + (0 if s == me else rcl[s])) * 8] for s in range(w)]
                dist.all_to_all(outs_d, self._views(self.send_dir, bank, [0 if d == me else c for d, c in enumerate(counts)], 8))
                ev[3].record(self.sb)
                self.hc.shard_unpack(rcl, self_bank=bank, stream=self.sb.cuda_stream)
                ev[4].record(self.sb)
                self.sent[bank].record(self.sb)      # (the bank is free again once its own chunks have been restaged)
        self.sa.synchronize()
        self.sb.synchronize()
        t = [0.0, 0.0, 0.0]
        for ev in marks:
            t[0] += ev[0].elapsed_time(ev[1]); t[1] += ev[2].elapsed_time(ev[3]); t[2] += ev[3].elapsed_time(ev[4])
        self.trace = {"rounds": rounds_all, "extract_ms": t[0], "exchange_ms": t[1], "restage_ms": t[2]}


class ShareReader(object):
    """Rank r's share of one file (jellyfish_b200.split.Share) read with pread, piece by piece, into two pinned host buffers:
    host memory stays bounded whatever the size of the file (the seam, read whole, holds the lines walked back in front of
    the share: one line for FASTA whose sequences are not wrapped).

    Piece i covers the bytes from the end of piece i - 1 to start + (i + 1) * piece_bytes (the last one to the end of the
    share), so every rank knows its number of pieces before it reads any.  A piece that is not the last one ends in front
    of a trailing run of '\\r', which then begins the next piece: a device feed that ends on '\\r' takes the run for a line
    end, where the byte behind it decides.  A run of CR_SLACK bytes or more there is refused (ValueError).

    records=True (FASTQ counted with -Q, whose feeds must end behind a whole record): a piece that is not the last one ends
    instead behind the last complete 4-line record in front of its nominal end, found on the reading thread, and the next
    piece starts there.  The nominal ends are then RECORD_SLACK (a quarter) of piece_bytes apart less, so that a piece is
    never longer than piece_bytes; a record that does not end in that last quarter is refused (ValueError).  The pieces
    still tile the share, so the newlines tallied over them are the share's.

    prefetch(i) reads piece i on a thread of its own, so that the disk or page-cache read overlaps the device work the
    caller enqueues meanwhile; read(i) then only waits for it."""

    CR_SLACK = 4096
    RECORD_SLACK = 4        # records=True: the last piece_bytes // RECORD_SLACK bytes of a nominal piece hold its record end

    def __init__(self, path, share, piece_bytes, records=False):
        from . import _lib
        self._lib = _lib.load()
        self.fmt = share.fmt
        self.share = share
        self.records = records
        self.slack = max(self.CR_SLACK, piece_bytes // self.RECORD_SLACK) if records else self.CR_SLACK
        self.piece = max(1, piece_bytes - self.slack)
        n = max(0, share.end - share.start)
        self.n_pieces = (n + self.piece - 1) // self.piece
        self.fd = os.open(path, os.O_RDONLY)
        self.bufs = [None, None]
        self.events = [None, None]
        self.next_off = share.start
        self._ahead = None                    # (piece, thread, [result or exception])
        # without a seam the share's first piece begins the file's parse (JFGPU_FILE_BEGIN with the format flag)
        self.first_begins = share.seam >= share.start

    def seam(self):
        """The seam's bytes (b"" when there is none)."""
        s = self.share
        return os.pread(self.fd, s.start - s.seam, s.seam) if s.seam < s.start else b""

    def _load(self, i):
        import ctypes as C
        b = i & 1
        if self.bufs[b] is None:
            p = self._lib.jfgpu_host_alloc(self.piece + self.slack)
            if not p:
                raise MemoryError("pinned host allocation failed")
            self.bufs[b] = p
        elif self.events[b] is not None:
            self.events[b].synchronize()          # the copy of piece i - 2 out of this buffer is done
        last = i == self.n_pieces - 1
        stop = self.share.end if last else self.share.start + (i + 1) * self.piece
        off = self.next_off
        view = (C.c_char * (stop - off)).from_address(self.bufs[b])
        got = os.preadv(self.fd, [view], off)
        if got != stop - off:
            raise IOError("short read of %d bytes at %d" % (stop - off, off))
        n = got
        if not last and self.records:
            n = self._record_end(view, n, stop)
        elif not last:
            tail = bytes(memoryview(view)[max(0, n - self.CR_SLACK):n])
            run = len(tail) - len(tail.rstrip(b"\r"))
            if run == len(tail):
                raise ValueError("a run of at least %d '\\r' bytes ends at byte %d, where the share is cut into pieces: "
                                 "count this file with --split files" % (run, stop))
            n -= run
        self.next_off = off + n
        return self.bufs[b], n, i == 0 and self.first_begins, last

    def _record_end(self, view, n, stop):
        """The length of the longest prefix of the n bytes read that ends behind a whole 4-line record (the piece starts on
        one): the last '\n' of the last `slack` bytes whose index in the piece is a multiple of 4."""
        import numpy as np
        a = np.frombuffer(view, dtype=np.uint8, count=n)
        step = 16 << 20
        lines = sum(int(np.count_nonzero(a[o:o + step] == 10)) for o in range(0, n, step))
        t0 = max(0, n - self.slack)
        at = np.flatnonzero(a[t0:] == 10)
        ends = at[(lines - len(at) + 1 + np.arange(len(at))) % 4 == 0]
        if not len(ends):
            raise ValueError("no FASTQ record ends in the %d bytes in front of byte %d, where the share is cut into pieces "
                             "(a record of more than %d bytes, or records of more than 4 lines): count this file with "
                             "--split files" % (n - t0, stop, self.slack))
        return t0 + int(ends[-1]) + 1

    def prefetch(self, i):
        """Start reading piece i (the pieces before it have been read) on a thread; nothing when i is past the last."""
        import threading
        if i >= self.n_pieces or self._ahead is not None:
            return
        box = []

        def run():
            try:
                box.append(self._load(i))
            except BaseException as ex:            # handed to read(i)
                box.append(ex)
        t = threading.Thread(target=run, daemon=True)
        self._ahead = (i, t, box)
        t.start()

    def read(self, i):
        """-> (host pointer, n, begin, end) of piece i; pieces are read in order.  The buffer stays untouched until piece i + 2
        is read or prefetched, which waits for the event release(i) records."""
        if self._ahead is not None:
            j, t, box = self._ahead
            t.join()
            self._ahead = None
            if j == i:
                if isinstance(box[0], BaseException):
                    raise box[0]
                return box[0]
        return self._load(i)

    def release(self, i, stream=None):
        """Piece i has been copied out (on `stream`; None: synchronously)."""
        if stream is None:
            self.events[i & 1] = None
            return
        ev = torch.cuda.Event()
        ev.record(stream)
        self.events[i & 1] = ev

    def close(self):
        if self._ahead is not None:
            self._ahead[1].join()
            self._ahead = None
        for p in self.bufs:
            if p:
                self._lib.jfgpu_host_free(p)
        self.bufs = [None, None]
        if self.fd >= 0:
            os.close(self.fd)
            self.fd = -1


def fastq_cuts_agree(tallies, world, device):
    """The FASTQ check of a split count: tallies = [(bytes, newlines) of this rank's share] per split FASTQ file, in the same
    file order on every rank.  Gathers every rank's tallies and returns True when every non-empty share of every file
    starts on a record (split.fastq_cuts_ok).  Every rank must call it."""
    from .split import fastq_cuts_ok
    if world == 1 or not tallies:
        return True
    mine = torch.tensor(tallies, dtype=torch.int64, device=device)
    every = [torch.empty_like(mine) for _ in range(world)]
    dist.all_gather(every, mine)
    every = [t.tolist() for t in every]
    return all(fastq_cuts_ok([every[r][f] for r in range(world)]) for f in range(len(tallies)))


def all_ranks_ok(ok, world, device):
    """True when `ok` holds on every rank (one all-reduce; every rank must call it)."""
    if world == 1:
        return bool(ok)
    t = torch.tensor([1 if ok else 0], dtype=torch.int64, device=device)
    dist.all_reduce(t, op=dist.ReduceOp.MIN)
    return bool(t.item())


def default_batch_bytes(k):
    """Text per exchange round of the key exchange.  Its three buffers (send, the second send bank, recv) take about
    8 * key_words * 1.25 bytes per batch byte each: 256 MB batches for k <= 64 (one or two key words), 64 MB for four-word
    keys (k > 64), whose 256 MB batches would take about 32 GB and leave no room for a wide shard of 2^30 slots (43 GB)
    on an 80 GB card."""
    return (64 << 20) if k is not None and k > 64 else (256 << 20)


class ShardedCounter(object):
    """hash_counter over `world` GPUs.  `size` is the GLOBAL table size (jellyfish count -s).

    Bloom structures (k <= 64): `bf_size` (count --bf-size, the GLOBAL expected number of k-mers; `bf_fp` its false positive
    rate) puts a prefilter in front of every shard, applied by the owner after the exchange; `bc` (count --bc) is the path of
    a counter written by `jellyfish bc`, loaded whole by every rank and applied by the sender before the exchange.  Both take
    the key exchange: the record exchange applies no filter.

    `disk` (count --disk) is a path prefix: the table does not double, and whenever this rank's shard is full it is written
    to a piece with `out_counter_len` bytes a count, zeroed, and counting goes on (`self.disk`, DiskPieces)."""

    def __init__(self, size, val_len=7, k=None, canonical=False, rank=0, world=1, device=0, reprobes=126,
                 batch_bytes=None, slack=1.25, exchange="auto", send_gb=None, bf_size=0, bf_fp=0.0, bc=None, disk=None,
                 out_counter_len=4, **engine_kw):
        from .engine import HashCounter
        if bf_size and bc:
            raise ValueError("Switches [--bf-size] and [--bc] conflict")
        if batch_bytes is None:
            batch_bytes = default_batch_bytes(k)
        self.rank, self.world = rank, world
        # -Q: every feed of FASTQ text must end behind a whole record (include/jfgpu.h: jfgpu_params.min_qual)
        self.qual = bool(engine_kw.get("min_qual"))
        self.hc = HashCounter(size, val_len, k=k, canonical=canonical, reprobes=reprobes, device=device,
                              shard_index=rank, n_shards=world, allow_regrow=(world == 1 and not disk), max_batch_bytes=batch_bytes,
                              bf_size=bf_size, bf_fp=bf_fp, **engine_kw)
        self.disk = DiskPieces(self.hc, disk, rank, out_counter_len) if disk else None
        if bc:
            # before the exchange form is chosen: the record exchange declines an engine with a Bloom structure
            self.hc.load_bloom_counter(bc)
        self.backend = EngineBackend(self.hc)
        self.batch_bytes = batch_bytes
        self.dev = torch.device("cuda", device)
        self.records = None
        if world > 1 and exchange in ("auto", "records"):
            rx = RecordExchange(self.hc, world, rank, self.dev, send_gb=send_gb)
            if rx.ok:
                self.records = rx
            elif exchange == "records":
                raise RuntimeError("the record exchange does not cover this table geometry")
            del rx
        if world > 1 and self.records is None:
            kw = self.hc.key_words
            # a batch of B bytes yields at most B k-mers, spread evenly over the owners by the hash
            self.capacity = int(batch_bytes / world * slack) + 65536
            self.send = torch.empty((world, self.capacity * kw), dtype=torch.int64, device=self.dev)
            self.recv = torch.empty((world, self.capacity * kw), dtype=torch.int64, device=self.dev)
            self.counts = torch.zeros(world, dtype=torch.int64, device=self.dev)
        self._host_stage = self._piece_stage = None
        self._send2 = self._counts2 = self._sa = None
        self._sam_out = None
        # host time of transcoding and routing the --sam pieces (jfgpu_sam_stage and the extraction, both synchronised;
        # one rank: transcoding and counting them)
        self.sam_device_s = 0.0
        # a dedicated (non-default) stream: its handle is passed to the engine so that kernels, tensor
        # ops and NCCL collectives are ordered on one stream (handle 0 would mean "engine stream")
        self.stream = torch.cuda.Stream(device=self.dev)

    def add_device_text(self, ptr, n, begin=True, end=True, fastq=False):
        """Device text, cut into exchange rounds.  fastq=True on an engine with -Q: the text is FASTQ that starts on a record
        and, unless it ends the file, ends behind one; the rounds are then cut behind whole records (record_bounds)."""
        if self.world == 1:
            self.hc.add_device_text(ptr, n, begin=begin, end=end)
            return
        torch.cuda.current_stream(self.dev).synchronize()     # the caller's text is complete
        budget = self.records.round_bytes if self.records is not None else self.batch_bytes
        bounds = self.record_bounds(ptr, n, budget) if fastq and self.qual else None
        if self.records is not None:
            self.records.add_device_text(ptr, n, begin, end, bounds)
            return
        with torch.cuda.stream(self.stream):
            self._add_device_text(ptr, n, begin, end, bounds)
        self.stream.synchronize()

    def record_bounds(self, ptr, n, budget):
        """[0, c_1, ..., c_m, n]: FASTQ text in device memory cut behind whole records into pieces of at most `budget` bytes
        (jfgpu_fastq_cuts: one pass over the text, one synchronisation)."""
        if not n:
            return [0]
        cuts, _ = self.hc.fastq_cuts(ptr, n, budget)
        return [0] + cuts + [n]

    def _add_device_text(self, ptr, n, begin, end, bounds=None):
        if bounds is None:
            bounds = [min(n, i * self.batch_bytes) for i in range((n + self.batch_bytes - 1) // self.batch_bytes + 1)] if n else [0]

        def extract(i, send, counts):
            if i + 1 >= len(bounds):              # (another rank has more rounds)
                return
            off, ln = bounds[i], bounds[i + 1] - bounds[i]
            if ln:
                if (ptr + off) % 16 and self._piece_stage is None:
                    self._piece_stage = [torch.empty(self.batch_bytes + 256, dtype=torch.uint8, device=self.dev) for _ in range(2)]
                src = aligned_text(ptr + off, ln, self._piece_stage[i & 1] if self._piece_stage else None)
                self.backend.extract_route((src, ln), begin and off == 0, end and off + ln >= n, send, self.capacity, counts)
        self._pipeline(len(bounds) - 1, extract)

    def _pipeline(self, rounds, extract):
        """Two-stage software pipeline: the extraction of batch i+1 (stream A) overlaps the NVLink
        exchange and the owner-side insertion of batch i (stream B).  Two send/count buffer sets.
        extract(i, send, counts) buckets batch i on stream A (nothing when this rank has no text for it)."""
        t = torch.tensor([rounds], dtype=torch.int64, device=self.dev)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        rounds_all = int(t.item())        # every rank takes part in every exchange
        if self._send2 is None:
            self._send2 = torch.empty_like(self.send)
            self._counts2 = torch.zeros_like(self.counts)
            self._sa = torch.cuda.Stream(device=self.dev)
        sends, cnts = (self.send, self._send2), (self.counts, self._counts2)
        sb = self.stream                    # stream B: exchange + insertion
        sa = self._sa                       # stream A: extraction
        sa.wait_stream(sb)
        done_extract = [torch.cuda.Event(), torch.cuda.Event()]
        done_use = [torch.cuda.Event(), torch.cuda.Event()]
        for ev in done_use:
            ev.record(sb)

        def launch_extract(i):
            with torch.cuda.stream(sa):
                sa.wait_event(done_use[i & 1])           # the buffers of batch i-2 have been sent
                cnts[i & 1].zero_()
                extract(i, sends[i & 1], cnts[i & 1])
                done_extract[i & 1].record(sa)

        if rounds_all:
            launch_extract(0)
        for i in range(rounds_all):
            sb.wait_event(done_extract[i & 1])
            nxt = (lambda j=i + 1: launch_extract(j)) if i + 1 < rounds_all else None
            exchange_and_insert(self.backend, self.world, sends[i & 1], cnts[i & 1], self.capacity, self.recv, before_payload=nxt)
            done_use[i & 1].record(sb)
        sa.synchronize()

    def add_host_text(self, hptr, n, begin=True, end=True):
        """Host memory (pinned) -> staged through a device buffer batch by batch."""
        if self.world == 1:
            import ctypes as C
            self.hc.add_text((C.c_void_p(hptr), n), begin=begin, end=end)
            return
        if self.records is not None:
            self.records.add_host_text(hptr, n, begin, end)
            return
        with torch.cuda.stream(self.stream):
            self._add_host_text(hptr, n, begin, end)
        self.stream.synchronize()

    def _add_host_text(self, hptr, n, begin, end):
        if self._host_stage is None:
            self._host_stage = torch.empty(self.batch_bytes + 256, dtype=torch.uint8, device=self.dev)
        from . import _lib
        lib = _lib.load()
        import ctypes as C
        off = 0
        rounds = (n + self.batch_bytes - 1) // self.batch_bytes
        t = torch.tensor([rounds], dtype=torch.int64, device=self.dev)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        for i in range(int(t.item())):
            ln = max(0, min(self.batch_bytes, n - off))
            self.counts.zero_()
            if ln:
                # host -> device on the working stream (asynchronous for pinned memory)
                if lib.jfgpu_memcpy_h2d(C.c_void_p(self._host_stage.data_ptr()), C.c_void_p(hptr + off), ln, C.c_void_p(self.stream.cuda_stream)):
                    raise RuntimeError("host to device copy failed")
                self.backend.extract_route((self._host_stage.data_ptr(), ln), begin and off == 0, end and off + ln >= n,
                                           self.send, self.capacity, self.counts)
            exchange_and_insert(self.backend, self.world, self.send, self.counts, self.capacity, self.recv)
            off += ln

    def piece_bytes(self):
        """The most text one exchange round takes: a piece of a streamed share is never longer."""
        return self.records.round_bytes if self.records is not None else self.batch_bytes

    def add_pieces(self, reader, tally=None):
        """Count a share of a file read piece by piece (ShareReader, pieces of at most piece_bytes()).  Every rank calls this
        once per file, also with a share that is empty: every rank takes part in every exchange round.  The copy to the device
        and the extraction of piece i + 1 run beside the exchange and insertion of piece i.  tally: a device int64 tensor
        the newlines of the share are added to (jfgpu_count_newlines)."""
        if self.world == 1:
            for i in range(reader.n_pieces):
                hptr, ln, begin, end = reader.read(i)
                reader.prefetch(i + 1)
                self.hc.add_text((hptr, ln), begin=begin, end=end, fmt=reader.fmt)
                reader.release(i)
            return
        torch.cuda.current_stream(self.dev).synchronize()
        if self.records is not None:
            self.records.add_pieces(reader, tally)
            return
        if self._piece_stage is None:
            self._piece_stage = [torch.empty(self.batch_bytes + 256, dtype=torch.uint8, device=self.dev) for _ in range(2)]
        from . import _lib
        import ctypes as C
        lib = _lib.load()

        def extract(i, send, counts):
            if i >= reader.n_pieces:
                return
            hptr, ln, begin, end = reader.read(i)
            dst = self._piece_stage[i & 1].data_ptr()
            st = torch.cuda.current_stream(self.dev)
            if ln and lib.jfgpu_memcpy_h2d(C.c_void_p(dst), C.c_void_p(hptr), ln, C.c_void_p(st.cuda_stream)):
                raise RuntimeError("host to device copy failed")
            reader.release(i, st)
            reader.prefetch(i + 1)            # (read while the exchange of the piece before and this extraction run)
            if tally is not None:
                self.hc.count_newlines(dst, ln, tally.data_ptr(), stream=st.cuda_stream)
            self.hc.extract_route(dst, ln, send.data_ptr(), self.capacity, counts.data_ptr(), begin=begin, end=end,
                                  stream=st.cuda_stream, fmt=reader.fmt)
        with torch.cuda.stream(self.stream):
            self._pipeline(reader.n_pieces, extract)
        self.stream.synchronize()

    def sam_piece_bytes(self):
        """Input bytes of a SAM / BAM piece.  Its FASTQ is at most twice the piece plus the line or record the engine carries
        in from the piece before (at most batch_bytes / 2), and it holds at most half as many k-mers as bytes: so the FASTQ
        of a piece holds no more k-mers than piece_bytes() of text."""
        return max(1, min(self.piece_bytes(), self.batch_bytes) // 2)

    def add_sam_pieces(self, reader, tolerant=False):
        """Count a SAM or BAM file, or a share of one, read piece by piece (jellyfish_b200.split_sam readers, pieces of at most
        sam_piece_bytes()).  Every rank calls this once per file, also with no pieces.  Each piece is transcoded into FASTQ
        of whole records (jfgpu_sam_stage) and routed as a FASTQ file of its own.  Piece i + 1 is read and inflated on the
        reader's thread while piece i is transcoded, routed and exchanged.  The record exchange also transcodes and extracts
        piece i + 1 while its stream B exchanges piece i; the key exchange does not: its pipeline stages piece i + 1 (host
        synchronous) between the count exchange and the payload exchange of piece i.  tolerant: a malformed piece (JFGPU_ERR_FORMAT, e.g. a BAM share whose
        record chain does not end at the next share's start) ends this reader's work, and False is returned; the other
        ranks go on with the exchange rounds.  Returns True otherwise."""
        from .engine import JellyfishError
        from . import _lib as L
        if self.world == 1:
            for i in range(reader.n_pieces):
                data, begin, end = reader.read(i)
                reader.prefetch(i + 1)
                t0 = time.perf_counter()
                self.hc.add_sam_text(data, begin=begin, end=end, bam=reader.bam)
                self.sam_device_s += time.perf_counter() - t0
                reader.release(i)
            return True
        torch.cuda.current_stream(self.dev).synchronize()
        if self._sam_out is None:
            self._sam_cap = 2 * (self.sam_piece_bytes() + self.batch_bytes // 2) + 64
            self._sam_out = [torch.empty(self._sam_cap, dtype=torch.uint8, device=self.dev) for _ in range(2)]
        ok = [True]

        def stage(i, st):
            out = self._sam_out[i & 1].data_ptr()
            if i >= reader.n_pieces or not ok[0]:
                return out, 0
            try:
                data, begin, end = reader.read(i)
                reader.prefetch(i + 1)       # (inflated while this piece is transcoded and the piece before is exchanged)
                n = self.hc.sam_stage(data, out, self._sam_cap, begin=begin, end=end, bam=reader.bam, stream=st.cuda_stream)
                reader.release(i)
            except JellyfishError as ex:
                if not tolerant or ex.code != L.ERR_FORMAT:
                    raise
                ok[0] = False
                return out, 0
            return out, n
        if self.records is not None:
            self.sam_device_s += self.records.add_sam_pieces(reader.n_pieces, stage)
            return ok[0]

        def extract(i, send, counts):
            t0 = time.perf_counter()
            ptr, n = stage(i, torch.cuda.current_stream(self.dev))
            if n:
                self.hc.extract_route(ptr, n, send.data_ptr(), self.capacity, counts.data_ptr(), begin=True, end=True,
                                      stream=torch.cuda.current_stream(self.dev).cuda_stream, fmt="fastq")
            self.sam_device_s += time.perf_counter() - t0
        with torch.cuda.stream(self.stream):
            self._pipeline(reader.n_pieces, extract)
        self.stream.synchronize()
        return ok[0]

    def set_op(self, op):
        """COUNT, PRIME or UPDATE on this rank (HashCounter.set_op: what is staged is drained under the operation before).
        Every rank switches at the same point of the exchange rounds: each add_* call returns once this rank has inserted,
        or restaged into its own record pool, everything it received, and a peer's records of the next operation only
        arrive through the next exchange round, which this rank enters after the switch."""
        self.hc.set_op(op)

    def done(self):
        return self.hc.done()

    def dump_shard(self, path, **kw):
        """Every rank writes `path.<rank>`: header (global size/matrix) + its sorted records."""
        return self.hc.dump("%s.%d" % (path, self.rank), **kw)


class DiskPieces(object):
    """`count --disk` on one rank: the spill hook of its engine `hc` writes the shard as it stands to piece
    `<prefix>.<rank>.<i>` (i = 0, 1, ...: `pieces`) with `out_counter_len` bytes a count, and the engine zeroes it and goes
    on counting.  No rank waits for another: each piece is a database of the GLOBAL geometry that holds only this shard's
    positions, so merging each rank's pieces and concatenating the results in rank order is the merge of all of them
    (write_output, concat_shards).  `spill_s`: the seconds spent writing pieces from inside the hook."""

    def __init__(self, hc, prefix, rank, out_counter_len=4):
        self.hc, self.disk, self.rank, self.out_counter_len = hc, prefix, rank, out_counter_len
        self.pieces = []
        self.spill_s = 0.0
        hc.set_spill(self._spill)

    def _write_piece(self, cmdline=()):
        """The table as it stands, every record, into the next piece."""
        path = piece_path(self.disk, self.rank, len(self.pieces))
        self.pieces.append(path)
        self.hc.dump(path, out_counter_len=self.out_counter_len, cmdline=cmdline)

    def _spill(self, hc):
        t0 = time.perf_counter()
        self._write_piece()
        self.spill_s += time.perf_counter() - t0

    def discard_pieces(self):
        """Delete the pieces written so far and number the next one 0 again: the table is about to be cleared and its input
        counted again (the fall-back of a failed cut check)."""
        for p in self.pieces:
            if os.path.exists(p):
                os.unlink(p)
        self.pieces = []

    def write_output(self, path, lower=0, upper=UINT64_MAX, cmdline=(), merge=True, unlink=True):
        """The end of a --disk count on this rank, after done().  A rank that never spilled dumps its shard to `path` with
        lower / upper, as without --disk.  A rank that spilled writes its table as one more piece; then, with `merge`, it
        merges its pieces into `path` with lower / upper applied to the sums (merge_pieces) and, with `unlink`, deletes them.
        merge=False: every piece stays and `path` is not written (nothing is merged; a rank that never spilled then writes
        its table as its only piece).  Returns the seconds spent merging."""
        if self.pieces or not merge:
            self._write_piece(cmdline)
        if not merge:
            return 0.0
        if len(self.pieces) == 0:
            self.hc.dump(path, lower=lower, upper=upper, out_counter_len=self.out_counter_len, cmdline=cmdline)
            return 0.0
        t0 = time.perf_counter()
        merge_pieces(self.pieces, path, self.hc.header(self.out_counter_len, cmdline), lower, upper)
        if unlink:
            for p in self.pieces:
                os.unlink(p)
        return time.perf_counter() - t0


class BloomBackend(object):
    """What the combination of Bloom counters across ranks needs from the engine; the CUDA engine implements it with kernels.
    A counter is n_words 32-bit words (16 positions each, two bits a position: hit, hit again) whose file body has n_bytes
    bytes (five positions a byte)."""

    n_words = n_bytes = 0

    def words(self):
        """int32 tensor of the counter's n_words words (read-only; on the device of the exchange)"""
        raise NotImplementedError

    def fold(self, words, first_word):
        """fold an int32 tensor of another counter's words into words [first_word, first_word + len(words))"""
        raise NotImplementedError

    def dump_range(self, first_byte, n_bytes, sink):
        """sink(bytes) with bytes [first_byte, first_byte + n_bytes) of the file body"""
        raise NotImplementedError


class _DeviceWords(object):
    """A device buffer the engine owns, seen by torch (CUDA array interface)."""

    def __init__(self, ptr, n):
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": "<i4", "data": (ptr, False), "version": 2}


class EngineBloomBackend(BloomBackend):
    """libjfgpu.so behind the seam: jfgpu_bloom_words / jfgpu_bloom_fold / jfgpu_bloom_dump_range of a BloomCounter."""

    def __init__(self, bc, dev):
        self.bc, self.dev = bc, dev

    def words(self):
        ptr, self.n_words = self.bc.words()
        self.n_bytes = self.bc.info()["nb_bytes"]
        return torch.as_tensor(_DeviceWords(ptr, self.n_words), device=self.dev)

    def fold(self, words, first_word):
        # on torch's current stream, behind the collective that delivered the words
        self.bc.fold(words.data_ptr(), first_word, words.numel(), stream=torch.cuda.current_stream(self.dev).cuda_stream)

    def dump_range(self, first_byte, n_bytes, sink):
        torch.cuda.current_stream(self.dev).synchronize()     # every fold is done
        self.bc.dump_range(first_byte, n_bytes, sink)


def bloom_slices(n_words, world):
    """[first_word, end_word) of every rank's slice of a counter: boundaries on the 5-word grid (80 positions, 16 bytes of
    the file body), the last slice ends at n_words."""
    units = (n_words + 4) // 5
    return [(min(5 * (units * r // world), n_words), min(5 * (units * (r + 1) // world), n_words)) for r in range(world)]


def bloom_byte_range(first_word, end_word, n_words, n_bytes):
    """The bytes of the file body that words [first_word, end_word) of a slice hold."""
    def to_byte(w):
        return n_bytes if w >= n_words else w // 5 * 16
    return to_byte(first_word), to_byte(end_word)


def bloom_reduce_scatter(backend, rank, world, piece_words=64 << 20):
    """Fold every rank's counter into the slice this rank owns (bloom_slices): a reduce-scatter made of all-to-alls of at
    most `piece_words` words per peer, so that it takes world * piece_words words of extra memory (256 MB per peer by
    default) rather than a second counter.  Returns this rank's (first_word, end_word)."""
    words = backend.words()
    sl = bloom_slices(words.numel(), world)
    longest = max(e - b for b, e in sl)
    pw = max(1, min(piece_words, longest))
    recv = torch.empty((world, pw), dtype=torch.int32, device=words.device)
    me0 = sl[rank][0]
    for p in range((longest + pw - 1) // pw):
        off = p * pw
        lens = [max(0, min(pw, e - b - off)) for b, e in sl]
        # this rank's own piece does not travel
        ins = [words[b + off:b + off + (0 if d == rank else lens[d])] for d, (b, e) in enumerate(sl)]
        rl = [0 if s == rank else lens[rank] for s in range(world)]
        outs = [recv[s, :rl[s]] for s in range(world)]
        if dist.get_backend() == "nccl":
            dist.all_to_all(outs, ins)
        else:
            flat = torch.empty(sum(rl), dtype=torch.int32, device=words.device)
            dist.all_to_all_single(flat, torch.cat(ins), output_split_sizes=rl, input_split_sizes=[x.numel() for x in ins])
            o = 0
            for s in range(world):
                outs[s].copy_(flat[o:o + rl[s]])
                o += rl[s]
        for s in range(world):
            if rl[s]:
                backend.fold(outs[s], me0 + off)
    return sl[rank]


class ShardedBloomCounter(object):
    """`jellyfish bc` over `world` GPUs (bc_main.cc:84-161): every rank builds a counter of its own text with the same k,
    size and false positive rate (so the same m, nb_hashes and matrices: the first draws of the reference's stream), then
    the counters are folded into one, rank r holding slice r (bloom_reduce_scatter), and every rank writes the bytes of its
    slice.  The combination is independent of the order of the hits, so the rank-ordered concatenation is the file one GPU
    (or the reference) writes for all the text."""

    def __init__(self, size, fpr=0.001, k=None, canonical=False, rank=0, world=1, device=0, piece_bytes=256 << 20):
        from .engine import BloomCounter
        self.rank, self.world = rank, world
        self.dev = torch.device("cuda", device)
        self.bc = BloomCounter(size, fpr, k=k, canonical=canonical, device=device)
        self.backend = EngineBloomBackend(self.bc, self.dev)
        self.piece_words = max(1, piece_bytes // 4)

    def add_files(self, paths):
        self.bc.add_files(paths)

    def combine(self):
        """-> (first_byte, n_bytes) of the file body this rank holds once every counter is folded in"""
        if self.world == 1:
            return 0, self.bc.info()["nb_bytes"]
        b, e = bloom_reduce_scatter(self.backend, self.rank, self.world, self.piece_words)
        first, end = bloom_byte_range(b, e, self.backend.n_words, self.backend.n_bytes)
        return first, end - first

    def dump_slice(self, path):
        """combine(), then `path.<rank>`: the body bytes of this rank's slice (no header)"""
        first, n = self.combine()
        out = "%s.%d" % (path, self.rank)
        with open(out, "wb") as f:
            self.backend.dump_range(first, n, f.write)
        return out

    def header(self, cmdline=()):
        return self.bc.header(cmdline)

    def close(self):
        self.bc.close()


def concat_bloom_slices(path, world, header, out=None):
    """header + the rank-ordered concatenation of the slice files `path.<rank>` (ShardedBloomCounter.dump_slice)."""
    from .engine import write_header
    out = out or path
    with open(out, "wb") as fo:
        write_header(fo, header)
        for r in range(world):
            with open("%s.%d" % (path, r), "rb") as fi:
                fo.write(fi.read())
    return out


def piece_path(prefix, rank, i):
    """Piece i of rank `rank` of a --disk count: `<prefix>.<rank>.<i>` (`<prefix>.<rank>` is the rank's shard file)."""
    return "%s.%d.%d" % (prefix, rank, i)


def merge_pieces(pieces, out, header, lower=0, upper=UINT64_MAX):
    """`jellyfish merge` of the pieces (databases of one geometry) into `out`, -L / -U applied to the sums, by the merge
    of the command built beside the library (the one `count --disk` ends with); `out` then gets `header` (the count's: the
    merge itself writes no `canonical` or `val_len`) in front of the merged records."""
    import shutil
    import subprocess
    from . import _lib
    from .engine import read_header, write_header
    tool = os.path.join(os.path.dirname(_lib.LIB_PATH), "jellyfish-b200")
    tmp = out + ".merging"
    cmd = [tool, "merge", "-o", tmp]
    if lower:
        cmd += ["-L", str(lower)]
    if upper != UINT64_MAX:
        cmd += ["-U", str(upper)]
    r = subprocess.run(cmd + list(pieces), stdout=subprocess.PIPE, stderr=subprocess.PIPE)
    if r.returncode != 0:
        raise RuntimeError("merging %s failed: %s" % (", ".join(pieces), r.stderr.decode(errors="replace").strip()))
    try:
        _, off = read_header(tmp)
        with open(tmp, "rb") as fi, open(out, "wb") as fo:
            write_header(fo, header)
            fi.seek(off)
            shutil.copyfileobj(fi, fo, 16 << 20)
    finally:
        os.unlink(tmp)
    return out


def concat_shards(path, world, out=None):
    """Rank-ordered concatenation of the shard files = the single-GPU database
    (positions of shard r all precede those of shard r+1)."""
    out = out or path
    with open(out, "wb") as fo:
        for r in range(world):
            with open("%s.%d" % (path, r), "rb") as fi:
                data = fi.read()
            hlen = int(data[:9])
            fo.write(data if r == 0 else data[9 + hlen:])
    return out
