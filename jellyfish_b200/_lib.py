"""ctypes binding of the C ABI in include/jfgpu.h (libjfgpu.so).

The library is built in-tree by `__graft_entry__.build()` (jellyfish_b200/csrc/Makefile).
There is no Python or CPU fallback: if the shared object is missing, importing this module
raises; if no CUDA device is present, `jfgpu_create` fails with a message saying so.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libjfgpu.so")

# every symbol include/jfgpu.h declares
SYMBOLS = [
    "jfgpu_create", "jfgpu_destroy", "jfgpu_last_error", "jfgpu_feed", "jfgpu_feed_device",
    "jfgpu_extract_route", "jfgpu_insert_keys", "jfgpu_clear", "jfgpu_set_op", "jfgpu_finish", "jfgpu_get_stats",
    "jfgpu_table_info_get", "jfgpu_dump", "jfgpu_lookup", "jfgpu_histogram",
    "jfgpu_reference_matrix", "jfgpu_synth_fasta_bytes", "jfgpu_synth_fasta_device",
    "jfgpu_host_alloc", "jfgpu_host_free", "jfgpu_memcpy_h2d", "jfgpu_kernel_launches", "jfgpu_version",
    "jfgpu_bloom_info_get", "jfgpu_bloom_load", "jfgpu_bloom_dump", "jfgpu_bloom_words", "jfgpu_bloom_fold", "jfgpu_bloom_dump_range",
    "jfgpu_set_spill", "jfgpu_shard_setup", "jfgpu_shard_round_bytes", "jfgpu_shard_extract", "jfgpu_shard_pack", "jfgpu_shard_unpack",
    "jfgpu_load_records", "jfgpu_query", "jfgpu_device_count", "jfgpu_seam", "jfgpu_seam_host", "jfgpu_count_newlines",
    "jfgpu_sam_stage", "jfgpu_fastq_cuts",
]

OK, ERR_ARG, ERR_CUDA, ERR_FULL, ERR_FORMAT, ERR_STATE, ERR_NOMEM, ERR_SINK = range(8)
FILE_BEGIN, FILE_END = 1, 2
FORMAT_SAM, FORMAT_BAM = 4, 8
FORMAT_FASTA, FORMAT_FASTQ = 16, 32


class Params(C.Structure):
    _fields_ = [
        ("struct_size", C.c_uint32), ("k", C.c_uint32), ("size", C.c_uint64),
        ("counter_len", C.c_uint32), ("max_reprobe", C.c_uint32), ("canonical", C.c_uint32),
        ("allow_regrow", C.c_uint32), ("device", C.c_int32), ("shard_index", C.c_uint32),
        ("n_shards", C.c_uint32), ("matrix_skip", C.c_uint32), ("bf_size", C.c_uint64),
        ("bf_fp", C.c_double), ("max_batch_bytes", C.c_uint64), ("pool_bytes", C.c_uint64),
        ("no_partition", C.c_uint32), ("part_min_mb", C.c_uint32), ("k2_mode", C.c_uint32), ("region_mb", C.c_uint32),
        ("bloom_counter", C.c_uint32), ("min_qual", C.c_uint32), ("reserved", C.c_uint64 * 2),
    ]


class TableInfo(C.Structure):
    _fields_ = [
        ("size", C.c_uint64), ("lsize", C.c_uint32), ("key_len", C.c_uint32), ("val_len", C.c_uint32),
        ("max_reprobe", C.c_uint32), ("matrix_r", C.c_uint32), ("matrix_c", C.c_uint32),
        ("matrix_identity", C.c_uint32), ("slot_bits", C.c_uint32), ("local_slots", C.c_uint64),
        ("table_bytes", C.c_uint64), ("matrix_columns", C.POINTER(C.c_uint64)),
        ("reprobes", C.POINTER(C.c_uint64)), ("part_regions", C.c_uint32), ("part_rec_bytes", C.c_uint32),
    ]


class Stats(C.Structure):
    _fields_ = [
        ("kmers", C.c_uint64), ("inserted", C.c_uint64), ("distinct", C.c_uint64), ("reprobes", C.c_uint64),
        ("overflowed", C.c_uint64), ("regrows", C.c_uint64), ("bytes", C.c_uint64), ("seconds_count", C.c_double),
        ("seconds_count_kernel", C.c_double), ("count_kernel_launches", C.c_uint64), ("seconds_drain", C.c_double),
        ("seconds_win_hist", C.c_double), ("seconds_win_scatter", C.c_double), ("seconds_win_insert", C.c_double),
    ]


class ShardBuffers(C.Structure):
    _fields_ = [
        ("send_pool", C.c_void_p), ("send_dir", C.c_void_p), ("send_arena_chunks", C.c_uint64),
        ("recv_pool", C.c_void_p), ("recv_dir", C.c_void_p), ("recv_seg_chunks", C.c_uint64),
    ]


class BloomInfo(C.Structure):
    _fields_ = [
        ("mode", C.c_uint32), ("nb_hashes", C.c_uint32), ("m", C.c_uint64), ("nb_bytes", C.c_uint64),
        ("matrix_r", C.c_uint32), ("matrix_c", C.c_uint32), ("matrix1", C.POINTER(C.c_uint64)), ("matrix2", C.POINTER(C.c_uint64)),
    ]


SINK_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_void_p, C.c_size_t)
SPILL_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_void_p)

_lib = None


def load():
    """Load libjfgpu.so (once) and declare the prototypes. Raises if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError("%s is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                          "(there is no CPU fallback)" % LIB_PATH)
    lib = C.CDLL(LIB_PATH)
    H = C.c_void_p
    lib.jfgpu_create.argtypes = [C.POINTER(Params), C.POINTER(H)]
    lib.jfgpu_create.restype = C.c_int
    lib.jfgpu_destroy.argtypes = [H]
    lib.jfgpu_destroy.restype = None
    lib.jfgpu_last_error.argtypes = [H]
    lib.jfgpu_last_error.restype = C.c_char_p
    lib.jfgpu_feed.argtypes = [H, C.c_void_p, C.c_size_t, C.c_uint32]
    lib.jfgpu_feed.restype = C.c_int
    lib.jfgpu_feed_device.argtypes = [H, C.c_void_p, C.c_size_t, C.c_uint32, C.c_void_p]
    lib.jfgpu_feed_device.restype = C.c_int
    lib.jfgpu_extract_route.argtypes = [H, C.c_void_p, C.c_size_t, C.c_uint32, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p]
    lib.jfgpu_extract_route.restype = C.c_int
    lib.jfgpu_insert_keys.argtypes = [H, C.c_void_p, C.c_uint64, C.c_void_p]
    lib.jfgpu_insert_keys.restype = C.c_int
    lib.jfgpu_set_op.argtypes = [H, C.c_uint32]
    lib.jfgpu_set_op.restype = C.c_int
    lib.jfgpu_clear.argtypes = [H]
    lib.jfgpu_clear.restype = C.c_int
    lib.jfgpu_finish.argtypes = [H, C.POINTER(Stats)]
    lib.jfgpu_finish.restype = C.c_int
    lib.jfgpu_get_stats.argtypes = [H, C.POINTER(Stats)]
    lib.jfgpu_get_stats.restype = C.c_int
    lib.jfgpu_table_info_get.argtypes = [H, C.POINTER(TableInfo)]
    lib.jfgpu_table_info_get.restype = C.c_int
    lib.jfgpu_dump.argtypes = [H, C.c_uint64, C.c_uint64, C.c_uint32, SINK_FN, C.c_void_p, C.POINTER(C.c_uint64)]
    lib.jfgpu_dump.restype = C.c_int
    lib.jfgpu_lookup.argtypes = [H, C.c_void_p, C.c_size_t, C.c_void_p]
    lib.jfgpu_lookup.restype = C.c_int
    lib.jfgpu_histogram.argtypes = [H, C.c_void_p, C.c_uint32]
    lib.jfgpu_histogram.restype = C.c_int
    lib.jfgpu_reference_matrix.argtypes = [C.c_uint32, C.c_uint32, C.c_uint32, C.c_void_p]
    lib.jfgpu_reference_matrix.restype = C.c_int
    lib.jfgpu_synth_fasta_bytes.argtypes = [C.c_uint64]
    lib.jfgpu_synth_fasta_bytes.restype = C.c_uint64
    lib.jfgpu_synth_fasta_device.argtypes = [C.c_int, C.c_void_p, C.c_uint64, C.c_uint64, C.c_uint64, C.POINTER(C.c_uint64), C.c_void_p]
    lib.jfgpu_synth_fasta_device.restype = C.c_int
    lib.jfgpu_host_alloc.argtypes = [C.c_size_t]
    lib.jfgpu_host_alloc.restype = C.c_void_p
    lib.jfgpu_host_free.argtypes = [C.c_void_p]
    lib.jfgpu_host_free.restype = None
    lib.jfgpu_memcpy_h2d.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]
    lib.jfgpu_memcpy_h2d.restype = C.c_int
    lib.jfgpu_kernel_launches.argtypes = []
    lib.jfgpu_kernel_launches.restype = C.c_uint64
    lib.jfgpu_version.argtypes = []
    lib.jfgpu_version.restype = C.c_char_p
    lib.jfgpu_bloom_info_get.argtypes = [H, C.POINTER(BloomInfo)]
    lib.jfgpu_bloom_info_get.restype = C.c_int
    lib.jfgpu_bloom_load.argtypes = [H, C.c_uint64, C.c_uint32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]
    lib.jfgpu_bloom_load.restype = C.c_int
    lib.jfgpu_bloom_dump.argtypes = [H, SINK_FN, C.c_void_p]
    lib.jfgpu_bloom_dump.restype = C.c_int
    lib.jfgpu_bloom_words.argtypes = [H, C.POINTER(C.c_void_p), C.POINTER(C.c_uint64)]
    lib.jfgpu_bloom_words.restype = C.c_int
    lib.jfgpu_bloom_fold.argtypes = [H, C.c_void_p, C.c_uint64, C.c_uint64, C.c_void_p]
    lib.jfgpu_bloom_fold.restype = C.c_int
    lib.jfgpu_bloom_dump_range.argtypes = [H, C.c_uint64, C.c_uint64, SINK_FN, C.c_void_p]
    lib.jfgpu_bloom_dump_range.restype = C.c_int
    lib.jfgpu_set_spill.argtypes = [H, SPILL_FN, C.c_void_p]
    lib.jfgpu_set_spill.restype = C.c_int
    lib.jfgpu_shard_setup.argtypes = [H, C.POINTER(ShardBuffers)]
    lib.jfgpu_shard_setup.restype = C.c_int
    lib.jfgpu_shard_round_bytes.argtypes = [H]
    lib.jfgpu_shard_round_bytes.restype = C.c_uint64
    lib.jfgpu_shard_extract.argtypes = [H, C.c_void_p, C.c_size_t, C.c_uint32, C.c_uint32, C.c_void_p]
    lib.jfgpu_shard_extract.restype = C.c_int
    lib.jfgpu_shard_pack.argtypes = [H, C.c_uint32, C.POINTER(C.c_uint64), C.c_void_p]
    lib.jfgpu_shard_pack.restype = C.c_int
    lib.jfgpu_shard_unpack.argtypes = [H, C.POINTER(C.c_uint64), C.c_uint32, C.c_void_p]
    lib.jfgpu_shard_unpack.restype = C.c_int
    lib.jfgpu_load_records.argtypes = [H, C.c_void_p, C.c_size_t, C.c_uint32]
    lib.jfgpu_load_records.restype = C.c_int
    lib.jfgpu_query.argtypes = [H, C.c_void_p, C.c_size_t, C.c_uint32, SINK_FN, C.c_void_p, C.POINTER(C.c_uint64)]
    lib.jfgpu_query.restype = C.c_int
    lib.jfgpu_seam.argtypes = [H, C.c_void_p, C.c_size_t, C.c_uint32, C.c_void_p]
    lib.jfgpu_seam.restype = C.c_int
    lib.jfgpu_seam_host.argtypes = [H, C.c_void_p, C.c_size_t, C.c_uint32]
    lib.jfgpu_seam_host.restype = C.c_int
    lib.jfgpu_count_newlines.argtypes = [H, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]
    lib.jfgpu_count_newlines.restype = C.c_int
    lib.jfgpu_fastq_cuts.argtypes = [H, C.c_void_p, C.c_size_t, C.c_uint32, C.c_uint64, C.POINTER(C.c_uint64), C.c_size_t,
                                     C.POINTER(C.c_size_t), C.POINTER(C.c_uint32), C.c_void_p]
    lib.jfgpu_fastq_cuts.restype = C.c_int
    lib.jfgpu_sam_stage.argtypes = [H, C.c_void_p, C.c_size_t, C.c_uint32, C.c_int, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t), C.c_void_p]
    lib.jfgpu_sam_stage.restype = C.c_int
    lib.jfgpu_device_count.argtypes = []
    lib.jfgpu_device_count.restype = C.c_int
    _lib = lib
    return lib
