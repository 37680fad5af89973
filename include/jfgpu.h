/* jfgpu.h -- C ABI of the H100 k-mer counting engine (libjfgpu.so).
 *
 * This is the drop-in boundary for the `jellyfish count` hot path.  The reference
 * (gmarcais/Jellyfish) has no FFI: its seam is the C++ template trio
 *   mer_overlap_sequence_parser  (include/jellyfish/mer_overlap_sequence_parser.hpp:61-114)
 *   hash_counter                 (include/jellyfish/hash_counter.hpp:50-172)
 *   dumper_t / sorted_dumper     (include/jellyfish/dumper.hpp:68-78, sorted_dumper.hpp:57-101)
 * driven by mer_counter_base::start (sub_commands/count_main.cc:152-184).  Each entry
 * point below names the reference interface it replaces.  Plain pointers and sizes
 * only; no C++ or torch types; no exception crosses the boundary: every call returns a
 * status (0 = OK) and jfgpu_last_error() gives the message.
 *
 * There is NO CPU fallback: every call that computes runs hand-written sm_90a CUDA.
 */
#ifndef JFGPU_H
#define JFGPU_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct jfgpu_engine* jfgpu_handle;

/* status codes */
enum {
  JFGPU_OK          = 0,
  JFGPU_ERR_ARG     = 1,  /* invalid argument / unsupported configuration           */
  JFGPU_ERR_CUDA    = 2,  /* CUDA runtime error (no device, launch failure, ...)    */
  JFGPU_ERR_FULL    = 3,  /* "Hash full": reference hash_counter.hpp:194-195         */
  JFGPU_ERR_FORMAT  = 4,  /* "Unsupported format": mer_overlap_sequence_parser.hpp:146 */
  JFGPU_ERR_STATE   = 5,  /* call sequence error                                    */
  JFGPU_ERR_NOMEM   = 6,  /* allocation failure (reference array::ErrorAllocation)   */
  JFGPU_ERR_SINK    = 7   /* the dump sink callback reported an error               */
};

/* feed flags */
enum {
  JFGPU_FILE_BEGIN = 1u,  /* first bytes of an input file: format is sniffed here    */
  JFGPU_FILE_END   = 2u,  /* last bytes of an input file: no k-mer spans the file end
                             (mer_overlap_sequence_parser.hpp:111)                  */
  /* Alignment records (count --sam, mer_overlap_sequence_parser.hpp:220-253).  Given with JFGPU_FILE_BEGIN, the file is read
   * in that form instead of being sniffed from its first byte, for all its feeds (a later feed may repeat the flag).  Every
   * record counts as a FASTQ read of its SEQ (ACGT in either case are bases, anything else an N) with its QUAL, FLAG ignored.
   * SAM: text; lines starting with '@' and blank lines are skipped, one '\r' in front of a '\n' ends the line; a QUAL of
   *   '*' gives every base the quality character 0x20.  jfgpu_feed and jfgpu_feed_device.
   * BAM: the INFLATED stream (magic "BAM\1", l_text, text, references, records; little-endian); quality character =
   *   phred + 33 (mod 256).  jfgpu_feed only.
   * An incomplete last line, header or record of a feed is carried to the next one.  A malformed record (fewer than 11
   * fields, SEQ and QUAL of different lengths, a BAM record or header cut short or with a bad magic) fails the feed with
   * JFGPU_ERR_FORMAT.  jfgpu_query, jfgpu_extract_route and jfgpu_shard_extract take neither flag (JFGPU_ERR_ARG). */
  JFGPU_FORMAT_SAM = 4u,
  JFGPU_FORMAT_BAM = 8u,
  /* Text that starts in the middle of a file (a share of one file split among ranks).  Given with JFGPU_FILE_BEGIN, the bytes
   * start at a line start of a file of this format and the first byte is not sniffed.  FASTA: the parser starts at a line
   * start (a share may begin on a sequence line).  FASTQ: the parser starts with a record's header line expected.  Taken by
   * jfgpu_feed, jfgpu_feed_device, jfgpu_extract_route, jfgpu_shard_extract, jfgpu_query and jfgpu_seam; the two exclude each
   * other and the SAM / BAM flags. */
  JFGPU_FORMAT_FASTA = 16u,
  JFGPU_FORMAT_FASTQ = 32u
};

/* operations of mer_counter_base (sub_commands/count_main.cc:133,152-184) */
enum { JFGPU_OP_COUNT = 0, JFGPU_OP_PRIME = 1, JFGPU_OP_UPDATE = 2 };

/* Constructor arguments: the union of hash_counter's constructor
 * (hash_counter.hpp:50-64: size, key_len, val_len, nb_threads, reprobe_limit) and the
 * switches of `jellyfish count` that act on the hot path
 * (sub_commands/count_main_cmdline.yaggo:4-112). */
typedef struct {
  uint32_t struct_size;    /* sizeof(jfgpu_params), for ABI evolution                */
  uint32_t k;              /* -m : mer length, 1..128.  Keys are 1 (k <= 32), 2 (k <= 64) or 4 (k > 64) 64-bit
                              words; k > 64 takes no Bloom structure (bf_size, bloom_counter) and at most 8 shards (the
                              key exchange only: jfgpu_extract_route / jfgpu_insert_keys), and is counted by direct
                              insertion into the wide slot form (slot_bits 320)   */
  uint64_t size;           /* -s : requested number of table slots (GLOBAL table);
                              rounded up to 2^l and clipped to 4^k exactly like
                              large_hash::array (large_hash_array.hpp:992-1002)      */
  uint32_t counter_len;    /* -c : "val_len" recorded in the header (default 7)       */
  uint32_t max_reprobe;    /* -p : reprobe limit before clipping (default 126)        */
  uint32_t canonical;      /* -C                                                      */
  uint32_t allow_regrow;   /* 1: double the table when full (hash_counter.hpp:200-238);
                              0: --disk: a full table goes to the spill hook (jfgpu_set_spill), JFGPU_ERR_FULL without one */
  int32_t  device;         /* CUDA device ordinal                                     */
  uint32_t shard_index;    /* this engine owns the slots whose top log2(n_shards)     */
  uint32_t n_shards;       /*   position bits equal shard_index (1 = whole table)     */
  uint32_t matrix_skip;    /* number of hash matrices to draw and discard first (so a
                              caller can reproduce a later point of the reference's
                              unseeded random() stream); normally 0                   */
  uint64_t bf_size;        /* --bf-size : expected number of k-mers, 0 = no filter     */
  double   bf_fp;          /* --bf-fp  (0 = the reference's default 0.01)              */
  uint64_t max_batch_bytes;/* device staging buffer size for jfgpu_feed (0 = default) */
  uint64_t pool_bytes;     /* HBM set aside for the k-mer record pool of the region-by-region
                              insertion (0 = 70% of the free memory, at most 64 GB)      */
  uint32_t no_partition;   /* 1: always insert straight into the table (random HBM access) */
  uint32_t part_min_mb;    /* tables of at least this many MB are filled region by region
                              (0 = default 256); tests use 1 to exercise that path on small tables */
  uint32_t k2_mode;        /* how the staged records reach the table (K2): 0 = default (shared-memory window
                              insert where the geometry allows it, else the L2 kernels), 1 = L2 kernels only,
                              2 = the generic L2 kernel only (no 32-bit specialisation), 3 = the window insert with
                              every group placed by the exact two-pass regroup (the fall-back of a window bucket
                              that overflows), 4 = the window insert with buckets of no slack, so that nearly every
                              group overflows one and falls back; for tests/benchmarks */
  uint32_t region_mb;      /* target size of a table region of the region-by-region insertion (0 = default 64); regions are made smaller when that lets a record fit 4 bytes */
  uint32_t bloom_counter;  /* 1: this engine builds a Bloom counter instead of a hash table -- `jellyfish bc`
                              (sub_commands/bc_main.cc:84-161): bf_size = expected number of k-mers (-s), bf_fp =
                              false positive rate (-f); `size`, `counter_len`, `max_reprobe` are ignored.  Feed text as
                              usual, then jfgpu_bloom_info_get / jfgpu_bloom_dump                                      */
  uint32_t min_qual;       /* -Q / --min-qual-char (the character) or --quality-start + --min-quality: bases whose quality character
                              is below it do not count (count_main.cc:234-256,326-329; mer_qual_iterator.hpp:64-92); 0 = off.
                              Text then has whole_sequence_parser semantics (a '\r' is an ordinary, window-resetting character);
                              FASTQ must be 4 lines per record, and a feed must end on a record boundary unless it ends the file */
  uint64_t reserved[2];
} jfgpu_params;

/* Description of the Bloom structure of an engine: what bc_main.cc:103-113 records in the "bloomcounter" header. */
typedef struct {
  uint32_t mode;           /* 0 none, 1 --bf-size prefilter, 2 Bloom counter being built, 3 loaded Bloom counter (--bc) */
  uint32_t nb_hashes;      /* bloom_base::k()                                          */
  uint64_t m;              /* bloom_base::m(): number of positions                     */
  uint64_t nb_bytes;       /* bytes jfgpu_bloom_dump streams (bloom_counter2: ceil(m/5)) */
  uint32_t matrix_r, matrix_c;     /* 64 x 2k                                          */
  const uint64_t* matrix1; /* matrix_c columns each; owned by the engine              */
  const uint64_t* matrix2;
} jfgpu_bloom_info;

/* What file_header::update_from_ary records (file_header.hpp:26-33). */
typedef struct {
  uint64_t size;           /* global number of slots, power of two                    */
  uint32_t lsize;          /* log2(size)                                              */
  uint32_t key_len;        /* 2k                                                      */
  uint32_t val_len;        /* -c                                                      */
  uint32_t max_reprobe;    /* clipped limit (large_hash_array.hpp:29-39,160)           */
  uint32_t matrix_r, matrix_c;
  uint32_t matrix_identity;/* 1 when the table is as large as the key space            */
  uint32_t slot_bits;      /* device slot width (32/64/128; 320 = the wide form of k > 64: a 64-bit head word
                              [counter | ready | reprobe+1] and the 4-word key); informational */
  uint64_t local_slots;    /* slots resident on this device (incl. overflow margin)   */
  uint64_t table_bytes;
  const uint64_t* matrix_columns; /* matrix_c columns (NULL when identity); owned by
                                     the engine, valid until the next regrow/destroy  */
  const uint64_t* reprobes;       /* max_reprobe+1 offsets (lib/storage.cc:13-41)      */
  uint32_t part_regions;   /* table regions of the region-by-region insertion (0 = direct insertion) */
  uint32_t part_rec_bytes; /* bytes of one staged k-mer record                                  */
} jfgpu_table_info;

typedef struct {
  uint64_t kmers;          /* k-mer windows emitted by the extractor                  */
  uint64_t inserted;       /* k-mers that reached the table (after filters)           */
  uint64_t distinct;       /* slots claimed                                           */
  uint64_t reprobes;       /* extra probes beyond the first, summed                   */
  uint64_t overflowed;     /* counter-field wrap events (exact: carried to side table)*/
  uint64_t regrows;        /* table doublings                                         */
  uint64_t bytes;          /* input bytes consumed                                    */
  double   seconds_count;  /* device time of whole feeds: copies + all kernels (CUDA events) */
  double   seconds_count_kernel; /* device time inside the fused count kernel alone,
                              summed over its launches (CUDA events on the launch stream) */
  uint64_t count_kernel_launches;
  double   seconds_drain;  /* device time of the region-by-region insertion passes (CUDA events) */
  double   seconds_win_hist, seconds_win_scatter, seconds_win_insert;   /* of which: the window kernels of K2 (jf_window.cuh),
                              CUDA events around their launches.  scatter: the bucket pass and the run starts; hist: the
                              exact placement of the groups that overflowed a window bucket (0 when none did); insert
                              includes the deferred-record kernel */
} jfgpu_stats;

/* -- life cycle: hash_counter ctor / dtor (hash_counter.hpp:50-68) ------------------ */
int  jfgpu_create(const jfgpu_params* params, jfgpu_handle* out);
void jfgpu_destroy(jfgpu_handle h);
const char* jfgpu_last_error(jfgpu_handle h);   /* h may be NULL: error of a failed create */

/* -- input: replaces mer_overlap_sequence_parser::produce + mer_iterator::operator++ +
 *    hash_counter::add for a whole buffer of FASTA text
 *    (mer_overlap_sequence_parser.hpp:88-114,161-185; mer_iterator.hpp:51-81;
 *     hash_counter.hpp:91-115).  Bytes of one file may be fed in any number of
 *    consecutive calls; state (header/sequence line, the k-1 base seam) is carried on
 *    the device.  `bytes` is HOST memory (pinned memory gives asynchronous copies). */
int  jfgpu_feed(jfgpu_handle h, const char* bytes, size_t n, uint32_t flags);
/* Same with the text already resident in device memory (16-byte aligned pointer).
 * `stream` is a cudaStream_t (NULL = the engine's own stream). */
int  jfgpu_feed_device(jfgpu_handle h, const void* dev_bytes, size_t n, uint32_t flags, void* stream);

/* -- SAM and BAM records turned into FASTQ without counting them (no reference analogue: the multi-GPU driver routes the
 *    FASTQ of a batch of whole records as a FASTQ file of its own, JFGPU_FILE_BEGIN | JFGPU_FILE_END | JFGPU_FORMAT_FASTQ,
 *    since no k-mer spans two reads).  The input is what jfgpu_feed (on_device = 0) or jfgpu_feed_device (on_device = 1,
 *    SAM only, 16-byte aligned) takes with JFGPU_FORMAT_SAM / _BAM: the same flags, the same carry of an incomplete last
 *    line, header field or record to the next call, the same JFGPU_ERR_FORMAT messages and byte offsets.  The FASTQ of the
 *    records completed by this call, "@\n SEQ \n+\n QUAL \n" each, is written to dev_out (device memory, any alignment)
 *    and *out_len receives its size; it is at most twice the bytes given plus those carried in, and JFGPU_ERR_ARG is returned
 *    when it would pass out_cap.  Nothing is counted and the text feeds are not disturbed: the staged file keeps its own
 *    carry, so jfgpu_feed, jfgpu_extract_route and jfgpu_shard_extract may run between two calls.  The call returns when the
 *    FASTQ is in dev_out; it runs after the work queued on `stream` (NULL = the engine's own stream). */
int  jfgpu_sam_stage(jfgpu_handle h, const void* bytes, size_t n, uint32_t flags, int on_device, void* dev_out, size_t out_cap,
                     size_t* out_len, void* stream);

/* -- the seam in front of a share of a file (no reference analogue: the reference reads every file whole).  Parse the text
 *    [dev_bytes, dev_bytes + n) and keep only what a feed leaves to the next one: the parser state and the last symbols
 *    (the k-1 base seam).  Nothing is counted: no table, route bucket or Bloom structure is touched and the statistics do not
 *    change.  The next call of jfgpu_feed, jfgpu_feed_device, jfgpu_extract_route or jfgpu_shard_extract without
 *    JFGPU_FILE_BEGIN continues from there, so that a seam of the text in front of a share followed by the share counts the
 *    k-mers of the share exactly as a feed of the whole file would.  Flags as for a feed (JFGPU_FILE_BEGIN with
 *    JFGPU_FORMAT_FASTA / _FASTQ in front of a share; JFGPU_FILE_END is refused, SAM and BAM too).  An engine with min_qual
 *    (-Q) is refused (JFGPU_ERR_ARG): its parser has other '\r' rules.  Synchronises `stream` (NULL = the engine's own).
 *    jfgpu_seam_host takes the text from HOST memory, as jfgpu_feed does. */
int  jfgpu_seam(jfgpu_handle h, const void* dev_bytes, size_t n, uint32_t flags, void* stream);
int  jfgpu_seam_host(jfgpu_handle h, const char* bytes, size_t n, uint32_t flags);
/* Add the number of '\n' bytes of [dev_bytes, dev_bytes + n) (device memory, any alignment) to *dev_count (a device uint64
 * the caller zeroes).  Stream-ordered on `stream` (NULL = the engine's own stream); the caller synchronises before reading
 * the count.  Used to check that the shares of a FASTQ file start on record boundaries. */
int  jfgpu_count_newlines(jfgpu_handle h, const void* dev_bytes, size_t n, uint64_t* dev_count, void* stream);
/* Cut FASTQ text (device memory, 16-byte aligned) behind whole 4-line records, so that every piece can be handed to a feed
 * of an engine with min_qual (-Q), which must end behind a record.  lines_mod4: the lines in front of dev_bytes (mod 4); a
 * record ends behind a '\n' in front of which the number of lines is a multiple of 4.  The cuts c_1 < c_2 < ... go to
 * `cuts` (host): c_i is the last record end at or before c_{i-1} + target (c_0 = 0), for as long as c_{i-1} + target < n.
 * So every piece [c_{i-1}, c_i) and the last one [c_m, n) holds at most `target` bytes; *n_cuts = m (at most
 * 2 * n / target + 1 when every record fits in target bytes).  *end_lines_mod4 (may be NULL): the lines (mod 4) at the end
 * of the text.  A record that does not end within target bytes of the piece it starts is JFGPU_ERR_FORMAT, as a record
 * larger than the staging batch of jfgpu_feed is; more than `cap` cuts is JFGPU_ERR_ARG.  Every byte is read once by one
 * kernel, and one CTA resolves the cuts; the call synchronises `stream` once (NULL = the engine's own stream). */
int  jfgpu_fastq_cuts(jfgpu_handle h, const void* dev_bytes, size_t n, uint32_t lines_mod4, uint64_t target, uint64_t* cuts,
                      size_t cap, size_t* n_cuts, uint32_t* end_lines_mod4, void* stream);

/* -- multi-GPU stages (no reference analogue; SURVEY.md section 8e) ------------------
 * Extract canonical k-mers from device-resident text and bucket them by owning shard
 * (top bits of the hash position).  dev_keys: n_shards * capacity packed keys
 * (8 bytes each for k<=32, 16 for k<=64, 32 for k<=128; word 0 first), bucket d at offset d*capacity;
 * 16-byte aligned for k > 64;
 * dev_counts: n_shards uint64 counters (accumulated; caller zeroes).
 * Returns JFGPU_ERR_FULL if a bucket overflowed (counts still exact, keys truncated).
 * With a caller stream and neither FILE flag the call is stream-ordered (no host synchronisation;
 * an overflow is then reported by jfgpu_finish). */
int  jfgpu_extract_route(jfgpu_handle h, const void* dev_bytes, size_t n, uint32_t flags,
                         void* dev_keys, uint64_t capacity, uint64_t* dev_counts, void* stream);
/* Insert n packed keys (as produced by jfgpu_extract_route) that this shard owns:
 * hash_counter::add for each (hash_counter.hpp:91-115).  With a caller stream the call is
 * stream-ordered (returns without synchronising).  A shard's table never doubles: keys that find
 * no slot are counted as failed and make jfgpu_finish return JFGPU_ERR_FULL ("Hash full"). */
int  jfgpu_insert_keys(jfgpu_handle h, const void* dev_keys, uint64_t n, void* stream);

/* Sharded counting, record exchange (the default for the geometries it covers -- k <= 21 with 32-bit slots; otherwise the
 * key exchange above).  K1 writes 4-byte records for the regions of the GLOBAL table into a SEND pool whose chunk arenas
 * belong to the owning shards: `jfgpu_shard_extract`.  `jfgpu_shard_pack` closes the open chunks and returns, per destination
 * d, the number of 8 KB chunks that sit at send_pool + (bank*n_shards + d)*send_arena_chunks*8192 (directory entries, 8 bytes
 * per chunk, at send_dir + the same index): the caller moves them (NCCL all-to-all) into the RECEIVE pool, source s at
 * recv_pool + s*recv_seg_chunks*8192 / recv_dir + s*recv_seg_chunks*8, and hands the counts to `jfgpu_shard_unpack`, which
 * turns them into records of this shard's own regions (restage_kernel); jfgpu_finish drains them into the table.
 * The pools are caller-owned device buffers (two send banks, so that the extraction of one round overlaps the exchange of
 * the previous one).  All calls are stream-ordered except jfgpu_shard_pack, which synchronises `stream`. */
typedef struct {
  void*    send_pool;          /* 2 * n_shards * send_arena_chunks * 8192 bytes */
  void*    send_dir;           /* 2 * n_shards * send_arena_chunks * 8 bytes    */
  uint64_t send_arena_chunks;
  void*    recv_pool;          /* n_shards * recv_seg_chunks * 8192 bytes        */
  void*    recv_dir;           /* n_shards * recv_seg_chunks * 8 bytes           */
  uint64_t recv_seg_chunks;    /* >= send_arena_chunks                           */
} jfgpu_shard_buffers;
int  jfgpu_shard_setup(jfgpu_handle h, const jfgpu_shard_buffers* buffers);   /* JFGPU_ERR_ARG: geometry not covered; with all
                                                                                pointers NULL the call only answers that question */
uint64_t jfgpu_shard_round_bytes(jfgpu_handle h);   /* text bytes one round (one bank) takes at most */
int  jfgpu_shard_extract(jfgpu_handle h, const void* dev_bytes, size_t n, uint32_t flags, uint32_t bank, void* stream);
int  jfgpu_shard_pack(jfgpu_handle h, uint32_t bank, uint64_t* chunks_per_dest /* [n_shards], host */, void* stream);
int  jfgpu_shard_unpack(jfgpu_handle h, const uint64_t* chunks_per_src /* [n_shards], host */, uint32_t self_bank, void* stream);
/*   self_bank 0/1: this shard's own chunks were not exchanged -- they are read from its arena of that send bank (which must
 *   stay untouched until `stream` has passed this call); any other value: they sit in the receive pool like everyone's. */

/* -- mer_counter_base's operation (sub_commands/count_main.cc:133,152-184): JFGPU_OP_COUNT adds
 *    (hash_counter::add), JFGPU_OP_PRIME inserts keys with count 0 (hash_counter::set, the first pass
 *    of `count --if`), JFGPU_OP_UPDATE adds only to keys already present (update_add, the second pass).
 *    Applies to the text fed after the call; drains pending work first. */
int  jfgpu_set_op(jfgpu_handle h, uint32_t op);

/* -- --disk (hash_counter::handle_full_ary without size doubling, hash_counter.hpp:187-192; count_main.cc:346-371): when the
 *    table is full and may not or cannot be doubled (allow_regrow = 0, or no device memory for twice the size), the engine
 *    calls `fn`, which writes the resident table out -- jfgpu_dump from inside the hook dumps the table as it stands --, then
 *    zeroes the table and goes on counting with the same geometry and matrix.  The caller merges the intermediate files
 *    (jellyfish merge / merge_files.cc:105-176).  Without a hook the same situations return JFGPU_ERR_FULL ("Hash full").
 *    On a shard (n_shards > 1) the hook is called when this shard is full, with no agreement between shards: jfgpu_dump
 *    from inside it writes this shard's own positions under the GLOBAL geometry, so every intermediate file of shard r is a
 *    database of the global size and matrix that holds positions of shard r only, and the merges of every shard's files,
 *    concatenated in shard order, are the merge of all of them.  The shard is zeroed (slots, overflow margin and counter-
 *    carry side table) and the keys that found no slot go into it.  With a hook, jfgpu_insert_keys and jfgpu_shard_unpack
 *    insert in slices of at most one failure group, each followed by a synchronisation of `stream` and, when keys failed,
 *    the drain of the pending region records and the spill: both return with every spill they caused complete.  A hook
 *    that returns non-zero ends the call with JFGPU_ERR_SINK. */
typedef int (*jfgpu_spill_fn)(void* ctx, jfgpu_handle h);
int  jfgpu_set_spill(jfgpu_handle h, jfgpu_spill_fn fn, void* ctx);

/* -- zero the table and the statistics, keep geometry and hash matrix: what the dumper's
 *    zero_blocks leaves behind (sorted_dumper.hpp:67-68,98-99) so the counter can be reused. */
int  jfgpu_clear(jfgpu_handle h);

/* -- hash_counter::done (hash_counter.hpp:169-172): drain all device work ------------ */
int  jfgpu_finish(jfgpu_handle h, jfgpu_stats* stats /* may be NULL */);
int  jfgpu_get_stats(jfgpu_handle h, jfgpu_stats* stats);
int  jfgpu_table_info_get(jfgpu_handle h, jfgpu_table_info* info);

/* -- output: replaces sorted_dumper::_dump/start + binary_writer::write
 *    (sorted_dumper.hpp:57-101, binary_dumper.hpp:36-40).  Streams this shard's records,
 *    ascending by (position, key), each = ceil(2k/8) little-endian key bytes followed by
 *    min(count, 2^(8*out_counter_len)-1) as out_counter_len little-endian bytes; only
 *    counts in [lower, upper] are emitted.  `sink` is called on the calling thread with
 *    consecutive byte ranges (whole records); a non-zero return aborts the dump. */
typedef int (*jfgpu_sink_fn)(void* ctx, const void* records, size_t nbytes);
int  jfgpu_dump(jfgpu_handle h, uint64_t lower, uint64_t upper, uint32_t out_counter_len,
                jfgpu_sink_fn sink, void* ctx, uint64_t* n_records /* may be NULL */);

/* -- lookup: array::get_val_for_key (large_hash_array.hpp:384-405).  keys: n packed
 *    k-mers in HOST memory (1, 2 or 4 uint64 words each for k <= 32, <= 64, <= 128; word 0 first); vals: n counts
 *    (0 when absent).  Keys not owned by this shard give 0. */
int  jfgpu_lookup(jfgpu_handle h, const uint64_t* keys, size_t n, uint64_t* vals);

/* -- a database back into a table: binary_query's database (binary_dumper.hpp:148-189) made resident.  `records` (HOST
 *    memory) holds whole records of a binary/sorted body, ceil(2k/8) little-endian key bytes then counter_len count bytes;
 *    any number of calls, each record's count is added.  The caller creates the engine with k = key_len/2 and `canonical`
 *    from the file's header, at least twice as many slots as records and allow_regrow = 1; the engine draws its own hash
 *    matrix (the database's matrix and size do not matter for look-ups).  The bytes go to the device through a pinned
 *    staging buffer in slices of at most 64 MB; a doubling during the load keeps the counts.  JFGPU_ERR_ARG: nbytes is
 *    not a whole number of records or counter_len is outside 1..8; JFGPU_ERR_NOMEM: the database does not fit. */
int jfgpu_load_records(jfgpu_handle h, const void* records, size_t nbytes, uint32_t counter_len);

/* -- query_from_sequence (sub_commands/query_main.cc:45-51): every k-mer of the text, in input order, as the line
 *    "MER COUNT\n" (MER in upper case, canonical when the engine is; COUNT 0 when absent).  Same text contract as jfgpu_feed
 *    (host memory, FILE_BEGIN / FILE_END, FASTA or 4-line FASTQ sniffed per file, no k-mer spans files; -Q does not
 *    apply).  `sink` is called on the calling thread with consecutive byte ranges of whole lines, in order; a non-zero
 *    return aborts the query (JFGPU_ERR_SINK).  *n_kmers (may be NULL) = lines written.  The table is not modified. */
int jfgpu_query(jfgpu_handle h, const char* bytes, size_t n, uint32_t flags,
                jfgpu_sink_fn sink, void* ctx, uint64_t* n_kmers);

/* -- histogram straight from the resident table (what `jellyfish histo` computes from
 *    the dump, sub_commands/histo_main.cc:33-45): hist[min(count,n_bins-1)]++ for every
 *    distinct k-mer of this shard.  hist: n_bins uint64 in HOST memory. */
int  jfgpu_histogram(jfgpu_handle h, uint64_t* hist, uint32_t n_bins);

/* -- Bloom structures in front of / instead of the table (count_main.cc:99-131,311-324; bc_main.cc) ---------------
 *    jfgpu_params.bf_size != 0 (with bloom_counter == 0) puts the one-pass prefilter of `count --bf-size` in front of the
 *    table: a k-mer reaches the table only when the filter has seen it before (bloom_filter.hpp:42-69).
 *    jfgpu_bloom_load puts a Bloom counter written by `jellyfish bc` in front of the table (count --bc,
 *    count_main.cc:191-206,110-120): `bytes` is the file body (five base-3 digits per byte), m / nb_hashes / the two
 *    64 x 2k matrices come from its header.  jfgpu_bloom_dump streams the body of the counter an engine created with
 *    bloom_counter = 1 has built (bloom_base::write_bits). */
int  jfgpu_bloom_info_get(jfgpu_handle h, jfgpu_bloom_info* info);
int  jfgpu_bloom_load(jfgpu_handle h, uint64_t m, uint32_t nb_hashes, const uint64_t* matrix1_cols, const uint64_t* matrix2_cols,
                      const void* bytes, size_t nbytes);
int  jfgpu_bloom_dump(jfgpu_handle h, jfgpu_sink_fn sink, void* ctx);   /* = jfgpu_bloom_dump_range over the whole body */

/* -- Bloom structures on the sharded path (no reference analogue: `jellyfish bc` and `count --bf-size/--bc` are one process)
 *    count --bc: every shard loads the whole counter (jfgpu_bloom_load) and jfgpu_extract_route drops a k-mer that fails it
 *    before bucketing it (filter_bc is a read-only test, count_main.cc:110-120).  The loaded form takes 1 bit per position:
 *    m / 8 bytes per shard, e.g. `bc -s 5G` at the default -f 0.001 (m = 14 bits per k-mer) 8.75 GB on every rank.
 *    count --bf-size: jfgpu_params.bf_size of a shard engine is the GLOBAL expected number of k-mers; each shard keeps a
 *    filter sized for ceil(bf_size / n_shards) of them (bloom_setup: bits and hash count as for one filter) in front of its
 *    own part of the table.  filter_bf (count_main.cc:122-133) drops the first occurrence of a k-mer, which needs one filter
 *    to see every occurrence: jfgpu_extract_route routes unfiltered and jfgpu_insert_keys applies the filter on the owner.
 *    The record exchange (jfgpu_shard_*) takes neither: jfgpu_shard_setup declines an engine with a Bloom structure and
 *    jfgpu_shard_extract returns JFGPU_ERR_STATE for one.
 *    `bc` across ranks: every rank builds a counter of its own text (bloom_counter = 1, the same k, size and fpr everywhere,
 *    so m, nb_hashes and both matrices agree).  A position of the counter is a saturating count min(2, hits)
 *    (bloom_counter2.hpp:56-107) held as two bits, (hit, hit again); combining two counters is order-independent:
 *    hit = hit_a | hit_b, again = again_a | again_b | (hit_a & hit_b). */
/* The counter's device words, read-only: ceil(m / 16) uint32, position p at bits 2*(p % 16) (hit) and 2*(p % 16) + 1 (hit
 * again) of word p / 16; positions >= m are 0.  Drains the engine's work first.  JFGPU_ERR_STATE: not a Bloom counter. */
int  jfgpu_bloom_words(jfgpu_handle h, void** dev_words, uint64_t* n_words);
/* Fold another counter of the same m, nb_hashes and matrices into this one: dev_words (device memory, n_words uint32 of
 * the layout above) are combined with words [first_word, first_word + n_words).  Stream-ordered on `stream` (NULL = the
 * engine's own stream): the caller synchronises it before reading or dumping the counter. */
int  jfgpu_bloom_fold(jfgpu_handle h, const void* dev_words, uint64_t first_word, uint64_t n_words, void* stream);
/* Bytes [first_byte, first_byte + n_bytes) of the file body bloom_base::write_bits writes (five base-3 digits per byte,
 * bloom_counter2.hpp:34-36; bc_main.cc:139).  first_byte must be a multiple of 16 (80 positions, 5 words), so that a range
 * starts on a word; the body has ceil(m / 5) bytes. */
int  jfgpu_bloom_dump_range(jfgpu_handle h, uint64_t first_byte, uint64_t n_bytes, jfgpu_sink_fn sink, void* ctx);

/* -- helpers ------------------------------------------------------------------------ */
/* The hash matrix the reference would draw as its (skip+1)-th matrix for a table of
 * 2^r slots and 2k = c key bits (rectangular_binary_matrix.cc:240-247 fed by the
 * unseeded glibc random() of lib/misc.cc:66-72).  cols: c uint64. Host-only arithmetic. */
int  jfgpu_reference_matrix(uint32_t r, uint32_t c, uint32_t skip, uint64_t* cols);
/* Synthetic FASTA of the shape jellyfish/generate_sequence.cc:119-149 writes (one
 * ">read1" record, 70 bases per line, iid uniform ACGT) generated directly in device
 * memory with a counter-based RNG.  Returns the number of bytes written in *n_bytes
 * (capacity must be >= jfgpu_synth_fasta_bytes(n_bases)). */
uint64_t jfgpu_synth_fasta_bytes(uint64_t n_bases);
int  jfgpu_synth_fasta_device(int device, void* dev_out, uint64_t capacity, uint64_t n_bases,
                              uint64_t seed, uint64_t* n_bytes, void* stream);
/* Pinned host memory for jfgpu_feed sources and dump sinks. */
void* jfgpu_host_alloc(size_t bytes);
void  jfgpu_host_free(void* p);
/* cudaMemcpyAsync host->device on `stream` (NULL = legacy default stream) for callers that have no
 * CUDA binding of their own; with memory from jfgpu_host_alloc the copy is asynchronous. */
int   jfgpu_memcpy_h2d(void* dev_dst, const void* host_src, size_t bytes, void* stream);
/* Number of CUDA devices visible to this process (0 without a device or a driver): lets a caller pick a CPU path. */
int   jfgpu_device_count(void);
/* Number of engine kernels launched so far by this process (bench "gpu_launches"). */
uint64_t jfgpu_kernel_launches(void);
const char* jfgpu_version(void);

#ifdef __cplusplus
}
#endif
#endif /* JFGPU_H */
