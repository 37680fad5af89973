"""Host-side mirror of the reference's counting interfaces, over the C ABI.

`HashCounter` follows the reference's `hash_counter` / SWIG `HashCounter`
(include/jellyfish/hash_counter.hpp:50-172, swig/hash_counter.i): construct with a size and a
value length, add k-mers, `done()`, read counts back, dump.  The difference is the unit of
work: k-mers are added a *buffer of FASTA text* at a time (`add_text`, `add_files`) because
parsing, canonicalisation, hashing and insertion run fused on the device.
"""
import ctypes as C
import json
import os
import time

from . import _lib as L

UINT64_MAX = (1 << 64) - 1


def text_flags(begin, end, fmt=None):
    """Feed flags of a piece of FASTA / FASTQ text.  fmt "fasta" or "fastq": the piece begins a share that starts at a line
    start in the middle of a file of that format (include/jfgpu.h: JFGPU_FORMAT_FASTA / _FASTQ); None: the format is sniffed
    from the first byte of the file."""
    f = (L.FILE_BEGIN if begin else 0) | (L.FILE_END if end else 0)
    if begin and fmt:
        f |= {"fasta": L.FORMAT_FASTA, "fastq": L.FORMAT_FASTQ}[fmt]
    return f


class JellyfishError(RuntimeError):
    """Raised for any non-zero status of the engine (reference: std::runtime_error / err::die)."""

    def __init__(self, code, msg):
        RuntimeError.__init__(self, msg)
        self.code = code


def reference_matrix(r, c, skip=0):
    """Columns of the hash matrix the reference draws (host arithmetic, no GPU needed)."""
    lib = L.load()
    cols = (C.c_uint64 * c)()
    rc = lib.jfgpu_reference_matrix(r, c, skip, cols)
    if rc:
        raise JellyfishError(rc, "invalid matrix dimensions")
    return list(cols)


def mer_to_int(s):
    """'ACGT...' -> 2-bit packed integer, first base most significant (mer_dna.hpp:525-542)."""
    v = 0
    for ch in s:
        v = (v << 2) | "ACGT".index(ch.upper())
    return v


def int_to_mer(v, k):
    return "".join("ACGT"[(v >> (2 * (k - 1 - i))) & 3] for i in range(k))


def canonical_int(v, k):
    rc = 0
    x = v
    for _ in range(k):
        rc = (rc << 2) | (3 - (x & 3))
        x >>= 2
    return min(v, rc)


class HashCounter(object):
    def __init__(self, size, val_len=7, k=None, canonical=False, reprobes=126, device=0,
                 shard_index=0, n_shards=1, allow_regrow=True, max_batch_bytes=0, matrix_skip=0,
                 pool_bytes=0, no_partition=False, part_min_mb=0, k2_mode=0, region_mb=0, bf_size=0, bf_fp=0.0,
                 bloom_counter=False, min_qual=0):
        if k is None:
            raise ValueError("k (mer length) is required")
        self._lib = L.load()
        self._h = C.c_void_p()
        p = L.Params()
        p.struct_size = C.sizeof(L.Params)
        p.k, p.size, p.counter_len, p.max_reprobe = k, size, val_len, reprobes
        p.canonical, p.allow_regrow, p.device = int(bool(canonical)), int(bool(allow_regrow)), device
        p.shard_index, p.n_shards, p.max_batch_bytes, p.matrix_skip = shard_index, n_shards, max_batch_bytes, matrix_skip
        p.pool_bytes, p.no_partition, p.part_min_mb = pool_bytes, int(bool(no_partition)), part_min_mb
        p.k2_mode, p.region_mb = k2_mode, region_mb
        p.bf_size, p.bf_fp, p.bloom_counter = bf_size, bf_fp, int(bool(bloom_counter))
        p.min_qual = ord(min_qual) if isinstance(min_qual, str) else int(min_qual)
        rc = self._lib.jfgpu_create(C.byref(p), C.byref(self._h))
        if rc:
            self._h = C.c_void_p()
            raise JellyfishError(rc, self._lib.jfgpu_last_error(None).decode())
        self.k = k
        self.canonical = bool(canonical)
        self.key_words = 4 if k > 64 else 2 if k > 32 else 1       # 64-bit words per key (jfgpu_lookup)
        self.n_shards = n_shards

    # -- plumbing ---------------------------------------------------------------------------
    def _check(self, rc):
        if rc:
            msg = self._lib.jfgpu_last_error(self._h).decode()
            cause = getattr(self, "_spill_error", None)
            if rc == L.ERR_SINK and cause is not None:
                self._spill_error = None
                raise JellyfishError(rc, "%s: %s" % (msg, cause)) from cause
            raise JellyfishError(rc, msg)

    def close(self):
        if getattr(self, "_h", None) and self._h.value:
            self._lib.jfgpu_destroy(self._h)
            self._h = C.c_void_p()
        self._spill_cb = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    # -- hash_counter interface -----------------------------------------------------------------
    def info(self):
        ti = L.TableInfo()
        self._check(self._lib.jfgpu_table_info_get(self._h, C.byref(ti)))
        d = {f: getattr(ti, f) for f, _ in L.TableInfo._fields_ if f not in ("matrix_columns", "reprobes")}
        d["matrix_columns"] = None if not ti.matrix_columns else [ti.matrix_columns[i] for i in range(ti.matrix_c)]
        d["reprobes"] = [ti.reprobes[i] for i in range(ti.max_reprobe + 1)]
        return d

    def size(self):
        return self.info()["size"]

    def val_len(self):
        return self.info()["val_len"]

    def add_text(self, data, begin=True, end=True, fmt=None):
        """Count every k-mer of a buffer of FASTA text held in host memory (bytes or a pointer/size pair).  fmt: see
        text_flags."""
        flags = text_flags(begin, end, fmt)
        if isinstance(data, tuple):
            ptr, n = data
        else:
            buf = bytes(data)
            ptr, n = C.cast(C.c_char_p(buf), C.c_void_p), len(buf)
        self._check(self._lib.jfgpu_feed(self._h, ptr, n, flags))

    def add_device_text(self, dev_ptr, n, begin=True, end=True, stream=None, sam=False, fmt=None):
        """Same with the text already in device memory (e.g. a torch uint8 tensor's data_ptr()); sam=True: SAM text."""
        flags = text_flags(begin, end, fmt) | (L.FORMAT_SAM if sam else 0)
        self._check(self._lib.jfgpu_feed_device(self._h, C.c_void_p(dev_ptr), n, flags, C.c_void_p(stream or 0)))

    def add_files(self, paths, chunk=64 << 20):
        """mer_counter_base::start over a list of files (count_main.cc:152-184)."""
        for path in paths:
            with open(path, "rb") as f:
                first = True
                cur = f.read(chunk)
                if not cur:
                    continue
                while True:
                    nxt = f.read(chunk)
                    self.add_text(cur, begin=first, end=not nxt)
                    first = False
                    if not nxt:
                        break
                    cur = nxt

    def add_sam_text(self, data, begin=True, end=True, bam=False):
        """Count the reads of SAM text, or (bam=True) of an inflated BAM stream, held in host memory (bytes or a pointer/size
        pair): each record's SEQ with its QUAL, as `count --sam` does (include/jfgpu.h: JFGPU_FORMAT_SAM / _BAM).  A file
        may come in any number of pieces, cut anywhere; `begin` and `end` mark its first and last."""
        flags = (L.FILE_BEGIN if begin else 0) | (L.FILE_END if end else 0) | (L.FORMAT_BAM if bam else L.FORMAT_SAM)
        if isinstance(data, tuple):
            ptr, n = data
        else:
            buf = bytes(data)
            ptr, n = C.cast(C.c_char_p(buf), C.c_void_p), len(buf)
        self._check(self._lib.jfgpu_feed(self._h, ptr, n, flags))

    def add_sam_files(self, paths, chunk=64 << 20):
        """`count --sam` over a list of files: SAM text, gzip'd SAM or BAM, told apart by their magic.  CRAM is refused."""
        import gzip
        for path in paths:
            with open(path, "rb") as raw:
                magic = raw.read(4)
            if magic.startswith(b"CRAM"):
                raise JellyfishError(L.ERR_FORMAT, "CRAM input is not supported ('%s')" % path)
            # (BGZF is multi-member gzip: the gzip module reads it whole)
            f = gzip.open(path, "rb") if magic[:2] == b"\x1f\x8b" else open(path, "rb")
            with f:
                cur = f.read(chunk)
                bam = cur[:4] == b"BAM\1"
                first = True
                while True:
                    nxt = f.read(chunk) if cur else b""
                    self.add_sam_text(cur, begin=first, end=not nxt, bam=bam)
                    first = False
                    if not nxt:
                        break
                    cur = nxt

    def sam_stage(self, data, out_ptr, out_cap, begin=True, end=True, bam=False, stream=None):
        """Turn SAM text or (bam=True) an inflated BAM stream into FASTQ without counting it (include/jfgpu.h:
        jfgpu_sam_stage).  data: bytes or a (pointer, size) pair in host memory, or ("device", pointer, size) for SAM text in
        device memory.  The FASTQ of the records this call completes goes to the device buffer at out_ptr (out_cap bytes);
        returns its size.  A file may come in any number of pieces, cut anywhere, as for add_sam_text."""
        flags = (L.FILE_BEGIN if begin else 0) | (L.FILE_END if end else 0) | (L.FORMAT_BAM if bam else L.FORMAT_SAM)
        on_device = isinstance(data, tuple) and len(data) == 3
        if on_device:
            ptr, n = C.c_void_p(data[1]), data[2]
        elif isinstance(data, tuple):
            ptr, n = C.c_void_p(data[0]) if isinstance(data[0], int) else data[0], data[1]
        else:
            buf = bytes(data)
            ptr, n = C.cast(C.c_char_p(buf), C.c_void_p), len(buf)
        out_len = C.c_size_t(0)
        self._check(self._lib.jfgpu_sam_stage(self._h, ptr, n, flags, int(on_device), C.c_void_p(out_ptr), out_cap, C.byref(out_len),
                                              C.c_void_p(stream or 0)))
        return out_len.value

    def seam(self, dev_ptr, n, fmt=None, begin=True, stream=None):
        """Parse device text [dev_ptr, dev_ptr + n) without counting it: the next feed without `begin` continues where it
        ends (include/jfgpu.h: jfgpu_seam).  The text in front of a share of a file, so that the share is counted as the
        whole file would count it."""
        self._check(self._lib.jfgpu_seam(self._h, C.c_void_p(dev_ptr), n, text_flags(begin, False, fmt), C.c_void_p(stream or 0)))

    def seam_text(self, data, fmt=None, begin=True):
        """seam() of text in host memory (bytes or a pointer/size pair): jfgpu_seam_host."""
        if isinstance(data, tuple):
            ptr, n = data
        else:
            buf = bytes(data)
            ptr, n = C.cast(C.c_char_p(buf), C.c_void_p), len(buf)
        self._check(self._lib.jfgpu_seam_host(self._h, ptr, n, text_flags(begin, False, fmt)))

    def count_newlines(self, dev_ptr, n, count_ptr, stream=None):
        """Add the '\\n' bytes of device text to the device uint64 at count_ptr (stream-ordered: jfgpu_count_newlines)."""
        self._check(self._lib.jfgpu_count_newlines(self._h, C.c_void_p(dev_ptr), n, C.c_void_p(count_ptr), C.c_void_p(stream or 0)))

    def fastq_cuts(self, dev_ptr, n, target, lines_mod4=0, stream=None):
        """Cut FASTQ text in device memory behind whole records into pieces of at most `target` bytes (include/jfgpu.h:
        jfgpu_fastq_cuts).  lines_mod4: the lines in front of the text (mod 4).  -> (the cuts, lines (mod 4) at the end); the
        pieces are [0, c_1), [c_1, c_2), ..., [c_m, n)."""
        cap = 2 * (n // target) + 2
        cuts = (C.c_uint64 * cap)()
        got, end = C.c_size_t(0), C.c_uint32(0)
        self._check(self._lib.jfgpu_fastq_cuts(self._h, C.c_void_p(dev_ptr), n, lines_mod4, target, cuts, cap, C.byref(got),
                                               C.byref(end), C.c_void_p(stream or 0)))
        return list(cuts[:got.value]), end.value

    def extract_route(self, dev_ptr, n, keys_ptr, capacity, counts_ptr, begin=True, end=True, stream=None, fmt=None):
        flags = text_flags(begin, end, fmt)
        self._check(self._lib.jfgpu_extract_route(self._h, C.c_void_p(dev_ptr), n, flags, C.c_void_p(keys_ptr),
                                                  capacity, C.c_void_p(counts_ptr), C.c_void_p(stream or 0)))

    def insert_keys(self, keys_ptr, n, stream=None):
        self._check(self._lib.jfgpu_insert_keys(self._h, C.c_void_p(keys_ptr), n, C.c_void_p(stream or 0)))

    # -- sharded counting, record exchange (include/jfgpu.h: jfgpu_shard_*) ----------------------------
    def shard_setup(self, send_pool, send_dir, send_arena_chunks, recv_pool, recv_dir, recv_seg_chunks):
        """Register the exchange buffers (device pointers).  False when the table geometry is not covered by the
        record exchange (the caller then uses extract_route / insert_keys)."""
        b = L.ShardBuffers(send_pool, send_dir, send_arena_chunks, recv_pool, recv_dir, recv_seg_chunks)
        rc = self._lib.jfgpu_shard_setup(self._h, C.byref(b))
        if rc == L.ERR_ARG:
            return False
        self._check(rc)
        return True

    def shard_round_bytes(self):
        return self._lib.jfgpu_shard_round_bytes(self._h)

    def shard_extract(self, dev_ptr, n, bank, begin=True, end=True, stream=None, fmt=None):
        flags = text_flags(begin, end, fmt)
        self._check(self._lib.jfgpu_shard_extract(self._h, C.c_void_p(dev_ptr), n, flags, bank, C.c_void_p(stream or 0)))

    def shard_pack(self, bank, stream=None):
        """Close the round: chunks per destination shard (synchronises the stream)."""
        n = self.n_shards
        counts = (C.c_uint64 * n)()
        self._check(self._lib.jfgpu_shard_pack(self._h, bank, counts, C.c_void_p(stream or 0)))
        return list(counts)

    def shard_unpack(self, counts, self_bank=None, stream=None):
        """counts: chunks received from every shard.  self_bank 0/1: this shard's own chunks are read from that send bank
        instead of the receive pool (they were not exchanged)."""
        arr = (C.c_uint64 * len(counts))(*counts)
        self._check(self._lib.jfgpu_shard_unpack(self._h, arr, 0xFFFFFFFF if self_bank is None else self_bank, C.c_void_p(stream or 0)))

    OP_COUNT, OP_PRIME, OP_UPDATE = 0, 1, 2

    def set_op(self, op):
        """COUNT (add), PRIME (insert with count 0) or UPDATE (add only to present keys): the two passes
        of `jellyfish count --if` (sub_commands/count_main.cc:288-295)."""
        self._check(self._lib.jfgpu_set_op(self._h, op))

    def set_spill(self, fn):
        """`count --disk` (include/jfgpu.h: jfgpu_set_spill): when the table is full and may not double (allow_regrow=False,
        or a shard), fn(self) is called to write it out -- normally self.dump(path, out_counter_len=...) without lower /
        upper, which dumps the table as it stands -- and the engine then zeroes the table and goes on counting with the same
        geometry and matrix.  The files it writes are merged at the end (`jellyfish merge`).  An exception raised by fn
        makes the engine call that filled the table fail with JellyfishError (ERR_SINK).  fn=None removes the hook."""
        def _hook(ctx, h):
            try:
                fn(self)
                return 0
            except BaseException as ex:        # (an exception cannot cross the C frames: it is raised by _check)
                self._spill_error = ex
                return 1
        cb = L.SPILL_FN(_hook) if fn is not None else L.SPILL_FN()
        self._check(self._lib.jfgpu_set_spill(self._h, cb, None))
        self._spill_cb = cb                     # (the engine calls it for as long as it lives)

    def clear(self):
        """Zero the table and statistics (same geometry and hash matrix)."""
        self._check(self._lib.jfgpu_clear(self._h))

    def done(self):
        """hash_counter::done -- drain the device, returns the statistics."""
        st = L.Stats()
        self._check(self._lib.jfgpu_finish(self._h, C.byref(st)))
        return {f: getattr(st, f) for f, _ in L.Stats._fields_}

    def stats(self):
        st = L.Stats()
        self._check(self._lib.jfgpu_get_stats(self._h, C.byref(st)))
        return {f: getattr(st, f) for f, _ in L.Stats._fields_}

    def get_many(self, mers):
        """Counts of a list of k-mers given as strings or packed ints (0 when absent)."""
        n = len(mers)
        kw = self.key_words
        keys = (C.c_uint64 * (n * kw))()
        for i, m in enumerate(mers):
            v = mer_to_int(m) if isinstance(m, str) else int(m)
            if self.canonical:
                v = canonical_int(v, self.k)
            for q in range(kw):
                keys[i * kw + q] = (v >> (64 * q)) & UINT64_MAX
        vals = (C.c_uint64 * n)()
        self._check(self._lib.jfgpu_lookup(self._h, keys, n, vals))
        return list(vals)

    def get(self, mer):
        v = self.get_many([mer])[0]
        return v if v else None

    __getitem__ = get

    def load_records(self, body, counter_len):
        """Add the records of a binary/sorted body (bytes, or a pointer/size pair in host memory): ceil(2k/8) key bytes
        then counter_len count bytes each."""
        if isinstance(body, tuple):
            ptr, n = body
        else:
            buf = bytes(body)
            ptr, n = C.cast(C.c_char_p(buf), C.c_void_p), len(buf)
        self._check(self._lib.jfgpu_load_records(self._h, ptr, n, counter_len))

    def query_text(self, data, begin=True, end=True, sink=None):
        """query_from_sequence (query_main.cc:45-51): the line "MER COUNT\n" for every k-mer of a buffer of FASTA / FASTQ
        text, in input order.  Returns the lines as bytes without a sink; with one, calls sink(bytes) with whole lines
        ("discard": the lines stay in the engine's pinned buffer) and returns the number of lines.  `query_bytes` is then
        the size of the output."""
        flags = (L.FILE_BEGIN if begin else 0) | (L.FILE_END if end else 0)
        if isinstance(data, tuple):
            ptr, n = data
        else:
            buf = bytes(data)
            ptr, n = C.cast(C.c_char_p(buf), C.c_void_p), len(buf)
        chunks = []

        self.query_bytes = 0

        def _sink(ctx, p, nb):
            self.query_bytes += nb
            if sink == "discard":
                return 0
            out = C.string_at(p, nb)
            if sink is None:
                chunks.append(out)
            else:
                sink(out)
            return 0

        cb = L.SINK_FN(_sink)
        nk = C.c_uint64(0)
        self._check(self._lib.jfgpu_query(self._h, ptr, n, flags, cb, None, C.byref(nk)))
        return b"".join(chunks) if sink is None else nk.value

    def query_files(self, paths, sink, chunk=64 << 20):
        """`query -s` over a list of files: sink(bytes) gets the lines of every k-mer, file after file; returns the number
        of lines."""
        n = 0
        for path in paths:
            with open(path, "rb") as f:
                first = True
                cur = f.read(chunk)
                while True:
                    nxt = f.read(chunk) if cur else b""
                    n += self.query_text(cur, begin=first, end=not nxt, sink=sink)
                    first = False
                    if not nxt:
                        break
                    cur = nxt
        return n

    def histogram(self, n_bins=10002):
        hist = (C.c_uint64 * n_bins)()
        self._check(self._lib.jfgpu_histogram(self._h, hist, n_bins))
        return list(hist)

    # -- Bloom structures (count --bf-size / --bc, `jellyfish bc`) ----------------------------------
    def bloom_info(self):
        bi = L.BloomInfo()
        self._check(self._lib.jfgpu_bloom_info_get(self._h, C.byref(bi)))
        d = {"mode": bi.mode, "nb_hashes": bi.nb_hashes, "m": bi.m, "nb_bytes": bi.nb_bytes}
        if bi.mode:
            d["matrix1"] = [bi.matrix1[i] for i in range(bi.matrix_c)]
            d["matrix2"] = [bi.matrix2[i] for i in range(bi.matrix_c)]
        return d

    def load_bloom_counter(self, path):
        """count --bc FILE (count_main.cc:191-206): filter by a Bloom counter written by `jellyfish bc`."""
        with open(path, "rb") as f:
            data = f.read()
        hlen = int(data[:9])
        hdr = json.loads(data[9:9 + hlen].rstrip(b"\0").decode())
        if hdr.get("format") != "bloomcounter":
            raise JellyfishError(L.ERR_FORMAT, "Invalid format '%s'. Expected 'bloomcounter'" % hdr.get("format"))
        if hdr["key_len"] != 2 * self.k:
            raise JellyfishError(L.ERR_ARG, "Invalid mer length in bloom filter")
        body = data[9 + hlen:]
        c = 2 * self.k
        m1 = (C.c_uint64 * c)(*hdr["matrix1"]["columns"])
        m2 = (C.c_uint64 * c)(*hdr["matrix2"]["columns"])
        self._check(self._lib.jfgpu_bloom_load(self._h, hdr["size"], hdr["nb_hashes"], m1, m2, body, len(body)))

    # -- dumper ------------------------------------------------------------------------------
    def dump_records(self, lower=0, upper=UINT64_MAX, out_counter_len=4, sink=None):
        """Sorted (position, key) record stream of this shard; returns bytes when no sink is given."""
        chunks = []

        def _sink(ctx, ptr, n):
            if sink == "discard":        # timing the device side of a dump: the bytes stay in the engine's pinned buffer
                return 0
            data = C.string_at(ptr, n)
            if sink is not None:
                sink(data)
            else:
                chunks.append(data)
            return 0

        cb = L.SINK_FN(_sink)
        nrec = C.c_uint64(0)
        self._check(self._lib.jfgpu_dump(self._h, lower, upper, out_counter_len, cb, None, C.byref(nrec)))
        return b"".join(chunks) if sink is None else nrec.value

    def header(self, out_counter_len=4, cmdline=()):
        """The file_header dictionary the reference writes (file_header.hpp:26-108)."""
        ti = self.info()
        m = {"r": ti["matrix_r"], "c": ti["matrix_c"], "identity": bool(ti["matrix_identity"])}
        if not ti["matrix_identity"]:
            m["columns"] = ti["matrix_columns"]
        sde = os.environ.get("SOURCE_DATE_EPOCH")
        return {
            "alignment": 8, "canonical": self.canonical, "cmdline": list(cmdline), "counter_len": out_counter_len,
            "exe_path": os.path.realpath(L.LIB_PATH), "format": "binary/sorted",
            "hostname": "hostname" if sde else os.uname().nodename, "key_len": ti["key_len"], "matrix1": m,
            "max_reprobe": ti["max_reprobe"], "pwd": "." if sde else os.getcwd(), "reprobes": ti["reprobes"],
            "size": ti["size"], "time": time.asctime(time.gmtime(int(sde))) if sde else time.asctime(),
            "val_len": ti["val_len"],
        }

    def dump(self, path, lower=0, upper=UINT64_MAX, out_counter_len=4, cmdline=()):
        """binary_dumper::dump -- header + sorted records (binary_dumper.hpp:62-69)."""
        with open(path, "wb") as f:
            write_header(f, self.header(out_counter_len, cmdline))
            return self.dump_records(lower, upper, out_counter_len, sink=f.write)


class BloomCounter(object):
    """`jellyfish bc` (sub_commands/bc_main.cc): a Bloom counter of the k-mers of some text, built on the device."""

    def __init__(self, size, fpr=0.001, k=None, canonical=False, device=0, max_batch_bytes=0):
        self.hc = HashCounter(1, 7, k=k, canonical=canonical, device=device, bf_size=size, bf_fp=fpr, bloom_counter=True,
                              max_batch_bytes=max_batch_bytes)
        self.k, self.canonical = k, bool(canonical)

    def close(self):
        self.hc.close()

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def add_files(self, paths):
        self.hc.add_files(paths)

    def add_text(self, data, begin=True, end=True, fmt=None):
        self.hc.add_text(data, begin=begin, end=end, fmt=fmt)

    def seam_text(self, data, fmt=None, begin=True):
        self.hc.seam_text(data, fmt=fmt, begin=begin)

    def info(self):
        return self.hc.bloom_info()

    def header(self, cmdline=()):
        bi = self.info()
        sde = os.environ.get("SOURCE_DATE_EPOCH")

        def mat(cols):
            return {"r": 64, "c": 2 * self.k, "identity": False, "columns": cols}
        return {
            "alignment": 8, "canonical": self.canonical, "cmdline": list(cmdline), "exe_path": os.path.realpath(L.LIB_PATH),
            "format": "bloomcounter", "hostname": "hostname" if sde else os.uname().nodename, "key_len": 2 * self.k,
            "matrix1": mat(bi["matrix1"]), "matrix2": mat(bi["matrix2"]), "nb_hashes": bi["nb_hashes"],
            "pwd": "." if sde else os.getcwd(), "size": bi["m"],
            "time": time.asctime(time.gmtime(int(sde))) if sde else time.asctime(),
        }

    def dump(self, path, cmdline=()):
        """header + filter.write_bits (bc_main.cc:113,139)."""
        with open(path, "wb") as f:
            write_header(f, self.header(cmdline))
            self.dump_range(0, self.info()["nb_bytes"], f.write)

    # -- combining counters across ranks (include/jfgpu.h: jfgpu_bloom_words / _fold / _dump_range) ------------------------
    def words(self):
        """-> (device pointer, number) of the counter's 32-bit words: position p at bits 2*(p % 16) (hit) and 2*(p % 16)+1
        (hit again) of word p // 16."""
        ptr, n = C.c_void_p(), C.c_uint64()
        self.hc._check(self.hc._lib.jfgpu_bloom_words(self.hc._h, C.byref(ptr), C.byref(n)))
        return ptr.value or 0, n.value

    def fold(self, dev_ptr, first_word, n_words, stream=None):
        """Fold n_words words of another counter (device memory) into words [first_word, first_word + n_words) of this one
        (stream-ordered)."""
        self.hc._check(self.hc._lib.jfgpu_bloom_fold(self.hc._h, C.c_void_p(dev_ptr), first_word, n_words, C.c_void_p(stream or 0)))

    def dump_range(self, first_byte, n_bytes, sink):
        """sink(bytes) with bytes [first_byte, first_byte + n_bytes) of the file body; first_byte a multiple of 16."""
        def _sink(ctx, ptr, n):
            sink(C.string_at(ptr, n))
            return 0
        cb = L.SINK_FN(_sink)
        self.hc._check(self.hc._lib.jfgpu_bloom_dump_range(self.hc._h, first_byte, n_bytes, cb, None))


def read_header(path):
    """-> (header dict, offset of the body) of a jellyfish file (generic_file_header.hpp:58-86)."""
    with open(path, "rb") as f:
        head = f.read(9)
        hlen = int(head)
        return json.loads(f.read(hlen).rstrip(b"\0").decode()), 9 + hlen


def load_database(path, device=0, size=None, max_batch_bytes=0):
    """A binary/sorted database (`jellyfish count` output) as a HashCounter resident on `device`: get_many, histogram,
    dump_records, query_text work on it.  The table gets its own hash matrix and at least twice as many slots as the
    file has records (`size` overrides that; the table doubles when it fills up, counts and all)."""
    hdr, off = read_header(path)
    if hdr.get("format") != "binary/sorted":
        raise JellyfishError(L.ERR_FORMAT, "Unsupported format '%s'. Must be a binary list." % hdr.get("format"))
    k = hdr["key_len"] // 2
    rec = (hdr["key_len"] + 7) // 8 + hdr["counter_len"]
    n_rec = (os.path.getsize(path) - off) // rec
    hc = HashCounter(size or max(2 * n_rec, 2), 7, k=k, canonical=hdr.get("canonical", False), device=device,
                     max_batch_bytes=max_batch_bytes)
    try:
        piece = max((256 << 20) // rec, 1) * rec
        with open(path, "rb") as f:
            f.seek(off)
            left = n_rec * rec
            while left:
                data = f.read(min(piece, left))
                hc.load_records(data, hdr["counter_len"])
                left -= len(data)
    except Exception:
        hc.close()
        raise
    return hc


def write_header(f, header):
    """generic_file_header::write (generic_file_header.hpp:88-111)."""
    h = json.dumps(header, sort_keys=True, separators=(",", ":"), ensure_ascii=False).encode()
    hlen = len(h)
    pad = (9 + hlen) % 8
    if pad:
        hlen += 8 - pad
    f.write(b"%09d" % hlen)
    f.write(h)
    if pad:
        f.write(b"\0" * (8 - pad))


class ReadMerFile(object):
    """Iterate the (mer, count) records of a binary/sorted database (swig/mer_file.i ReadMerFile)."""

    def __init__(self, path):
        with open(path, "rb") as f:
            data = f.read()
        hlen = int(data[:9])
        self.header = json.loads(data[9:9 + hlen].rstrip(b"\0").decode())
        self.body = data[9 + hlen:]
        self.k = self.header["key_len"] // 2
        self.key_bytes = (self.header["key_len"] + 7) // 8
        self.counter_len = self.header["counter_len"]

    def __iter__(self):
        rec = self.key_bytes + self.counter_len
        b = self.body
        for i in range(0, len(b) - rec + 1, rec):
            key = int.from_bytes(b[i:i + self.key_bytes], "little")
            yield int_to_mer(key, self.k), int.from_bytes(b[i + self.key_bytes:i + rec], "little")
