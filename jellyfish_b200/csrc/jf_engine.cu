// jf_engine.cu -- C-ABI implementation (include/jfgpu.h) of the H100 k-mer counting engine.
// Host orchestration only: every byte of the hot path is processed by the kernels in
// jf_kernels.cuh.  There is no CPU fallback; without a CUDA device every call fails.
#include <cuda_runtime.h>
#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <string>
#include <type_traits>
#include <utility>
#include <vector>

#include "../../include/jfgpu.h"
#include "host/jf_matrix.hpp"
#include "jf_kernels.cuh"
#include "jf_extract.cuh"
#include "jf_window.cuh"
#include "jf_dump.cuh"
#include "jf_shard.cuh"
#include "jf_query.cuh"
#include "jf_wide.cuh"
#include "jf_bloom.cuh"
#include "jf_sam.cuh"
#include "jf_newline.cuh"

using namespace jfk;

static std::atomic<unsigned long long> g_launches(0);
static thread_local std::string g_create_error;

#define JF_LAUNCHED() g_launches.fetch_add(1, std::memory_order_relaxed)

namespace {

constexpr unsigned SHARD_RESERVED_SMS = 16;
constexpr uint32_t SAM_FLAGS = JFGPU_FORMAT_SAM | JFGPU_FORMAT_BAM;
constexpr uint32_t TEXT_FLAGS = JFGPU_FORMAT_FASTA | JFGPU_FORMAT_FASTQ;
constexpr uint64_t WIN_DEF_CAP = (uint64_t)16 << 20;   // deferred records per group of the window form of K2   // SMs K1 leaves to NCCL while an exchange runs beside it

unsigned ceil_log2(uint64_t x) { unsigned l = 0; while(l < 64 && ((uint64_t)1 << l) < x) ++l; return l; }
unsigned bitsize(uint64_t x) { unsigned b = 0; while(x) { ++b; x >>= 1; } return b ? b : 1; }

// Owners of the engine's CUDA resources.  Each is move-only and empty while it holds nothing; what it holds is released
// when it is reset, reassigned or destroyed.  An allocation or creation that fails leaves it empty.
struct DevBuf {
  void* p = nullptr; size_t bytes = 0;
  DevBuf() = default;
  DevBuf(DevBuf&& o) noexcept : p(o.p), bytes(o.bytes) { o.p = nullptr; o.bytes = 0; }
  DevBuf& operator=(DevBuf&& o) noexcept { if(this != &o) { reset(); std::swap(p, o.p); std::swap(bytes, o.bytes); } return *this; }
  ~DevBuf() { reset(); }
  // (the old buffer is freed first: the old and the new one are never held at once)
  cudaError_t alloc(size_t n) { reset(); const cudaError_t c = n ? cudaMalloc(&p, n) : cudaSuccess; if(c == cudaSuccess) bytes = n; else p = nullptr; return c; }
  void reset() { if(p) cudaFree(p); p = nullptr; bytes = 0; }
  template<typename T> T* as() const { return reinterpret_cast<T*>(p); }
};

template<typename T> struct HostBuf {            // pinned host memory
  T* p = nullptr;
  HostBuf() = default;
  HostBuf(const HostBuf&) = delete;
  HostBuf(HostBuf&& o) noexcept : p(o.p) { o.p = nullptr; }
  HostBuf& operator=(HostBuf&& o) noexcept { if(this != &o) { reset(); std::swap(p, o.p); } return *this; }
  ~HostBuf() { reset(); }
  cudaError_t alloc(size_t bytes) { reset(); const cudaError_t c = cudaHostAlloc((void**)&p, bytes, cudaHostAllocDefault); if(c) p = nullptr; return c; }
  void reset() { if(p) cudaFreeHost(p); p = nullptr; }
  operator T*() const { return p; }
};

struct Event {
  cudaEvent_t ev = nullptr;
  Event() = default;
  Event(Event&& o) noexcept : ev(o.ev) { o.ev = nullptr; }
  ~Event() { reset(); }
  cudaError_t create(unsigned flags) { reset(); const cudaError_t c = cudaEventCreateWithFlags(&ev, flags); if(c) ev = nullptr; return c; }
  void reset() { if(ev) cudaEventDestroy(ev); ev = nullptr; }
  operator cudaEvent_t() const { return ev; }
};

struct Stream {
  cudaStream_t s = nullptr;
  Stream() = default;
  Stream(const Stream&) = delete;
  ~Stream() { if(s) cudaStreamDestroy(s); }
  cudaError_t create() { const cudaError_t c = cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking); if(c) s = nullptr; return c; }
  operator cudaStream_t() const { return s; }
};

// A member of a group for make_all: a buffer of `arg` bytes, or an event created with flags `arg`
template<typename O> struct Need {
  O& o; size_t arg;
  cudaError_t make() const {
    if constexpr(std::is_same<O, Event>::value) return o.create((unsigned)arg);
    else return o.alloc(arg);
  }
};
template<typename O> Need<O> need(O& o, size_t arg) { return Need<O>{o, arg}; }

// Make a group of resources all or nothing, in order.  When one fails, every member is reset, the error state is cleared
// and the error returned; so any one member tells whether the whole group is there.
template<typename... O> cudaError_t make_all(Need<O>... m) {
  cudaError_t c = cudaSuccess;
  (void)(((c = m.make()) == cudaSuccess) && ...);
  if(c != cudaSuccess) { (m.o.reset(), ...); cudaGetLastError(); }
  return c;
}

// byte-indexed tables of a GF(2) matrix: entry [b*256+v] = product with the vector whose
// byte b equals v (reference column order: bit i selects columns[c-1-i],
// rectangular_binary_matrix.hpp:223-261)
std::vector<uint64_t> build_lut(const jfb::gf2_matrix& m, unsigned nbytes) {
  std::vector<uint64_t> lut((size_t)nbytes * 256, 0);
  const unsigned c = m.c(), r = m.r();
  for(unsigned b = 0; b < nbytes; ++b) {
    uint64_t col[8];
    for(unsigned j = 0; j < 8; ++j) {
      unsigned i = 8 * b + j;
      if(i >= c) col[j] = 0;
      else if(m.is_identity()) col[j] = i < r ? ((uint64_t)1 << i) : 0;
      else col[j] = m[c - 1 - i];
    }
    for(unsigned v = 0; v < 256; ++v) {
      uint64_t x = 0;
      for(unsigned j = 0; j < 8; ++j) if(v & (1u << j)) x ^= col[j];
      lut[(size_t)b * 256 + v] = x;
    }
  }
  return lut;
}

struct Table {
  unsigned lsize = 0, local_lsize = 0, max_reprobe = 0, rbits = 1, fbits = 1, slot_bits = 32, hb = 0;
  uint64_t size = 0, local_size = 0, margin = 0, local_slots = 0, ovf_size = 0;
  // slots [materialized, local_size) are zero in meaning but not in memory (table_zero, table_materialize)
  uint64_t materialized = 0;
  jfb::gf2_matrix M, Minv;
  DevBuf slots, lut, inv_lut, ovf_keys, ovf_vals, lut11;
  DevBuf win_state;              // while materialized < local_size: one state per window (jf_kernels.cuh, WIN_LAZY ...)
  uint64_t prow[8] = {0,0,0,0,0,0,0,0}; unsigned n_prow = 0; bool hash_fast = false;
  std::vector<uint64_t> reprobes;
  size_t bytes() const { return (size_t)local_slots * (slot_bits / 8); }
};

}  // namespace

struct PartState {
  uint32_t P = 0, region_bits = 0, rec_bytes = 0, cap = 0, flush_min = 0, stage_bytes = 0, n_chunks = 0, margin = 0, arena_chunks = 0, n_arenas = 0;
  DevBuf pool, dir, order, pool_next, cta_chunk, cta_fill, spill_keys, spill_counts, spill_n, hist, start, cursor, unit_cursor;   // (hist: region_recs)
  uint64_t spill_cap = 0;
  // window form of K2 (jf_window.cuh)
  DevBuf w_start, w_cursor, w_cnt, w_rec, w_def_pos[2], w_def_high[2], w_def_n;    // (two deferred lists, w_def_n: their two lengths)
  DevBuf w_flag;                 // [PMAX] overflow flag of every group of a drain (a group that needed the exact placement)
  uint64_t w_rec_cap = 0, w_def_cap = 0;
  uint64_t bound_chunks = 0;     // host-side upper bound of the chunks in use in any one arena
  bool pending = false;          // records sit in the pool
};

// Sharded counting, record exchange (jf_shard.cuh): the send pool (global regions, one chunk arena per owning shard, two
// banks) and the receive pool live in buffers the caller registers (they are the NCCL send / receive buffers).
struct ShardState {
  bool on = false;
  uint32_t P = 0, sbits = 0, own_regions = 0, split_lg = 0, owner_shift = 0;
  uint64_t arena_chunks = 0, seg_chunks = 0;
  uint8_t* send_pool = nullptr; uint2* send_dir = nullptr; uint8_t* recv_pool = nullptr; uint2* recv_dir = nullptr;
  DevBuf pool_next[2], cta_chunk, cta_fill;
  HostBuf<unsigned int> h_counts;
};

struct BloomState {
  uint32_t mode = BLOOM_NONE, k = 0;
  uint64_t m = 0, inv = 0, n_words = 0;
  bool drawn = false;              // the two hash matrices have been drawn (lazily: after the --if pass, count_main.cc:288-321)
  jfb::gf2_matrix M1, M2;
  std::vector<uint64_t> cols1, cols2;
  DevBuf bits, locks, lut1, lut2;
};

struct jfgpu_engine {
  Stream cs, hs;                  // (first, so that they are destroyed last)
  jfgpu_params p;
  PartState part;
  ShardState sh;
  BloomState bloom;
  int device = 0;
  unsigned k = 0, kw = 1, nbytes = 0, shard_bits = 0;
  int n_sm = 132;
  jfb::glibc_random rng;
  Table tab;
  DevBuf stats, carry[2], fail_keys[2], fail_counts[2];
  uint64_t fail_cap = 0, fail_group = 0;    // failure list entries; records per group of a careful drain
  int carry_cur = 0, fail_cur = 0;
  HostBuf<unsigned long long> h_stats;      // mirror of `stats`
  // staging for host feeds
  size_t batch_bytes = 0;
  DevBuf stage[2]; Event ev_copied[2], ev_done[2];
  int stage_cur = 0;
  uint8_t stage_look[2] = {0, 0};           // look-ahead byte staged behind a batch that ends in '\r' (run_staged)
  // per-batch scratch
  DevBuf nlA, nlB, cntA, cntB, tstate; uint64_t scratch_tiles = 0;
  int format = 0;                 // 0 = FASTA, 1 = FASTQ: format of the file being fed
  // -Q on FASTQ: a batch must end on a record boundary (the qualities of a read are looked up two lines further down);
  // lines seen so far in the file (mod 4) and the incomplete last record of the previous feed
  uint32_t q_lines = 0; std::string q_tail;
  // --disk: what hash_counter::handle_full_ary does when the table cannot double (hash_counter.hpp:187-192): the caller's
  // hook dumps the resident table (jfgpu_dump from inside the hook), the engine zeroes it and goes on counting
  jfgpu_spill_fn spill_fn = nullptr; void* spill_ctx = nullptr; bool in_spill = false; uint64_t spills = 0;
  uint32_t op = 0;                // JFGPU_OP_*
  // bookkeeping
  bool in_file = false;
  uint64_t bytes_fed = 0, regrows = 0;
  double count_ms = 0;
  unsigned eff_val_len = 7;
  Event ev_t0, ev_t1;
  std::string err;
  std::vector<uint64_t> matrix_cols_host;   // for jfgpu_table_info_get
  std::vector<Event> kev;                   // event pairs around count_kernel launches
  size_t kev_used = 0;
  double kernel_ms = 0; uint64_t kernel_launches = 0;
  double drain_ms = 0; Event ev_d0, ev_d1;
  int count_smem = 0;
  // CUDA events around the window kernels of a drain: [4 per group] hist begin, scatter begin, insert begin, insert end
  std::vector<Event> wev; size_t wev_used = 0;
  double win_ms[3] = { 0, 0, 0 };
  // failure counter watched one group behind (hash_counter::add -> handle_full_ary), without draining the stream
  HostBuf<unsigned long long> h_watch; Event ev_watch[2];
  // jfgpu_query: two sets of per-batch buffers (the lines of batch i are copied out while batch i+1 is looked up)
  bool querying = false;
  struct QueryBufs {
    DevBuf keys, vals, cnt, off, out;
    HostBuf<unsigned long long> h_off;      // copy of `off` (entry n_tiles: the batch's total)
    HostBuf<uint32_t> h_cnt;                // copy of `cnt`
    uint64_t n_tiles = 0;
    Event ev_front, ev_fmt;
  } qb[2];
  HostBuf<uint8_t> q_host[2]; Event ev_qcopy[2];
  uint64_t q_tiles_cap = 0; int q_cur = 0;
  // jfgpu_seam: the ordered extraction runs into scratch that nobody reads (only the carry it leaves matters)
  bool seaming = false;
  DevBuf seam_keys, seam_cnt;
  DevBuf fq_scratch;                        // jfgpu_fastq_cuts
  // SAM / BAM input (jf_sam.cu): the form of the file being fed (0 = FASTA / FASTQ text, 1 = SAM, 2 = BAM), the buffers of a
  // batch (made at the first such file; one of each: a batch is transcoded and read back before the next is staged) and what
  // a feed leaves to the next one
  struct SamState {
    uint32_t form = 0;
    size_t in_cap = 0;                              // input bytes of a batch: its FASTQ, at most twice as long, is one K1 batch
    DevBuf out, scratch, res, offs, tail_dev;       // FASTQ, kernel scratch, jfsam::Result, BAM record offsets, device carry
    HostBuf<jfsam::Result> h_res; HostBuf<uint32_t> h_offs;
    std::string tail;                               // host feeds: the incomplete last line, or the cut BAM header field or record
    size_t tail_dev_len = 0;                        // device feeds: bytes of the incomplete last line in tail_dev
    uint32_t bam_phase = 0, bam_refs = 0;           // BAM walk: which header field comes next, references left
    uint64_t bam_skip = 0;                          // bytes of header text or reference name still to pass over
    uint64_t done_off = 0;                          // bytes of the file in front of the next batch (messages)
  } sam;
  // jfgpu_sam_stage: the file being staged keeps its own SamState (swapped into `sam` for the length of a call), so that the
  // feeds and routings between two stage calls do not reset its carry; a batch's FASTQ is appended to the caller's buffer
  SamState sam_staged;
  uint8_t* stage_out = nullptr;
  size_t stage_out_cap = 0, stage_out_len = 0;
};

namespace {

int fail(jfgpu_engine* e, int code, const std::string& msg) {
  if(e) e->err = msg; else g_create_error = msg;
  return code;
}
#define CUDA_OK(e, call) do { cudaError_t _c = (call); if(_c != cudaSuccess) \
  return fail(e, JFGPU_ERR_CUDA, std::string(#call) + ": " + cudaGetErrorString(_c)); } while(0)

TableDev table_dev(const jfgpu_engine* e, const Table& t) {
  TableDev d;
  memset(&d, 0, sizeof(d));
  d.slots = t.slots.p;
  d.local_mask = t.local_size - 1;
  d.local_lsize = t.local_lsize;
  d.lsize = t.lsize;
  d.shard_index = e->p.shard_index;
  d.kbits = 2 * e->k;
  d.rbits = t.rbits;
  d.fbits = t.fbits;
  d.max_reprobe = t.max_reprobe;
  d.op = e->op;
  d.ovf_keys = t.ovf_keys.as<unsigned long long>();
  d.ovf_vals = t.ovf_vals.as<unsigned long long>();
  d.ovf_mask = t.ovf_size - 1;
  d.stats = e->stats.as<unsigned long long>();
  d.fail_keys = e->fail_keys[e->fail_cur].as<uint64_t>();
  d.fail_counts = e->fail_counts[e->fail_cur].as<uint64_t>();
  d.fail_cap = e->fail_cap;
  return d;
}

// Geometry of a table of 2^lsize GLOBAL slots -- large_hash_array.hpp:150-173,29-39.
// `reprobe_limit` is -p for the first table and the CLIPPED limit of the previous table after a doubling: the reference
// hands ary_->max_reprobe() to the new array (hash_counter.hpp:205-209), so a limit clipped by a tiny table never grows back.
int table_setup(jfgpu_engine* e, Table& t, unsigned lsize, const jfb::gf2_matrix& M, unsigned reprobe_limit) {
  const unsigned kbits = 2 * e->k;
  t.lsize = lsize;
  t.size = (uint64_t)1 << lsize;
  t.local_lsize = lsize - e->shard_bits;
  t.local_size = (uint64_t)1 << t.local_lsize;
  t.hb = kbits > lsize ? kbits - lsize : 0;
  unsigned limit = kbits > lsize ? reprobe_limit : 0;
  // reprobes[0] = 1, reprobes[i] = i(i+1)/2 (lib/storage.cc:13-41); clip so that reprobes[limit] < size
  auto rp = [](unsigned i) -> uint64_t { return i == 0 ? 1 : tri(i); };
  while(limit >= 1 && rp(limit) >= t.size) --limit;
  t.max_reprobe = limit;
  t.reprobes.resize(limit + 1);
  for(unsigned i = 0; i <= limit; ++i) t.reprobes[i] = rp(i);
  t.rbits = bitsize(limit + 1);
  t.fbits = t.hb + t.rbits;
  // the narrowest slot that keeps at least 8 counter bits, so that only counts beyond ~250 need the carry side table; a
  // 128-bit slot also takes key fields of 121..127 bits (k = 61..64 in tables of at most 2^14 slots), whose 1..7-bit counter
  // carries into the side table on nearly every increment (it has at least 2^20 entries, such a table at most 2^14 slots)
  if(e->kw == 4) {                 // four-word keys: the wide form, the whole key beside a head word (jf_device.cuh, SB_WIDE)
    t.fbits = t.rbits + 1;         // the head's low bits: reprobe+1 and READY
    t.slot_bits = SB_WIDE;
  } else if(t.fbits <= 22) t.slot_bits = 32;
  else if(t.fbits <= 56) t.slot_bits = 64;
  else if(t.fbits <= 127) t.slot_bits = 128;
  else return fail(e, JFGPU_ERR_ARG, "key too long for this table size (k=" + std::to_string(e->k) + ", " + std::to_string(t.size) +
                                     " slots: a key field of " + std::to_string(t.fbits) + " bits, at most 127 fit a slot)");
  if(e->kw == 2 && t.slot_bits == 32) t.slot_bits = 64;
  t.margin = limit ? tri(limit) : 0;
  t.local_slots = t.local_size + t.margin + 8;
  t.M = M;
  t.Minv = M.pseudo_inverse();
  if(t.slots.alloc(t.bytes()) != cudaSuccess) {
    cudaGetLastError();
    char buf[128]; snprintf(buf, sizeof(buf), "Failed to allocate %zu bytes of device memory", t.bytes());
    return fail(e, JFGPU_ERR_NOMEM, buf);
  }
  // counter-carry side table: one entry per slot whose counter field wrapped; sized with the table
  t.ovf_size = (uint64_t)1 << 20;
  while(t.ovf_size < ((uint64_t)1 << 26) && t.ovf_size * 64 < t.local_size) t.ovf_size <<= 1;
  CUDA_OK(e, t.ovf_keys.alloc(t.ovf_size * 8));
  CUDA_OK(e, t.ovf_vals.alloc(t.ovf_size * 8));
  std::vector<uint64_t> l1 = build_lut(t.M, e->nbytes), l2 = build_lut(t.Minv, e->nbytes);
  CUDA_OK(e, t.lut.alloc(l1.size() * 8));
  CUDA_OK(e, t.inv_lut.alloc(l2.size() * 8));
  CUDA_OK(e, cudaMemcpyAsync(t.lut.p, l1.data(), l1.size() * 8, cudaMemcpyHostToDevice, e->cs));
  CUDA_OK(e, cudaMemcpyAsync(t.inv_lut.p, l2.data(), l2.size() * 8, cudaMemcpyHostToDevice, e->cs));
  // fast hash tables: 2k <= 44 -> four 11-bit chunks; entries = low 32 bits of the partial products,
  // position bits 32.. come from parity rows
  t.hash_fast = false; t.n_prow = 0;
  for(unsigned i = 0; i < 8; ++i) t.prow[i] = 0;            // (unused rows must be zero: K1 evaluates a fixed number of them)
  std::vector<uint32_t> l11;
  if(e->kw == 1 && kbits <= 44 && lsize <= 40) {
    l11.assign(4 * 2048, 0);
    auto colsel = [&](unsigned i) -> uint64_t {       // contribution of key bit i
      if(i >= t.M.c()) return 0;
      if(t.M.is_identity()) return i < t.M.r() ? ((uint64_t)1 << i) : 0;
      return t.M[t.M.c() - 1 - i];
    };
    for(unsigned tb = 0; tb < 4; ++tb)
      for(unsigned v = 0; v < 2048; ++v) {
        uint64_t x = 0;
        for(unsigned j = 0; j < 11; ++j) if(v & (1u << j)) x ^= colsel(tb * 11 + j);
        l11[tb * 2048 + v] = (uint32_t)x;
      }
    for(unsigned ob = 32; ob < lsize; ++ob) {
      uint64_t row = 0;
      for(unsigned i = 0; i < kbits; ++i) if((colsel(i) >> ob) & 1) row |= (uint64_t)1 << i;
      t.prow[t.n_prow++] = row;
    }
    CUDA_OK(e, t.lut11.alloc(l11.size() * 4));
    CUDA_OK(e, cudaMemcpyAsync(t.lut11.p, l11.data(), l11.size() * 4, cudaMemcpyHostToDevice, e->cs));
    t.hash_fast = true;
  }
  CUDA_OK(e, cudaStreamSynchronize(e->cs));     // the host vectors are about to go out of scope
  return JFGPU_OK;
}

// Zero a table (slots and counter-carry side table) on the compute stream.  `lazy`: slots [0, local_size) are zero in
// meaning only (materialized = 0, every window WIN_LAZY).  The next drain, window form, writes every window without reading
// it; the overflow margin past local_size, which deferred probes reach, is zeroed in memory as always.
int table_zero(jfgpu_engine* e, Table& t, bool lazy) {
  const size_t sb = t.slot_bits / 8, from = lazy ? (size_t)t.local_size * sb : 0;
  CUDA_OK(e, cudaMemsetAsync((uint8_t*)t.slots.p + from, 0, t.bytes() - from, e->cs));
  if(lazy) {
    const size_t n_win = (size_t)(t.local_size >> WIN_LG) * 4;
    if(!t.win_state.p) CUDA_OK(e, t.win_state.alloc(n_win));
    CUDA_OK(e, cudaMemsetAsync(t.win_state.p, 0, n_win, e->cs));
  }
  CUDA_OK(e, cudaMemsetAsync(t.ovf_keys.p, 0, t.ovf_size * 8, e->cs));
  CUDA_OK(e, cudaMemsetAsync(t.ovf_vals.p, 0, t.ovf_size * 8, e->cs));
  t.materialized = lazy ? 0 : t.local_size;
  return JFGPU_OK;
}

// Zero in memory the slots of a lazily zeroed table that no drain has written yet.  Every path that reads or updates
// slots other than the write-only window drain passes here first: part_drain (L2 and rehash forms, spill list),
// jfgpu_finish (and so lookup, histogram, dump, max_count and set_op), direct insertion by K1, insert_keys_into and
// jfgpu_shard_unpack (the record exchange therefore drains with loads, as before).  The
// window drain calls it itself before it returns, also when it stops for a regrow, so collect never sees such a table.
int table_materialize(jfgpu_engine* e, Table& t, cudaStream_t st) {
  if(t.materialized >= t.local_size) return JFGPU_OK;
  const uint64_t w0 = t.materialized >> WIN_LG;       // (a region boundary; the windows K1 put in memory keep their data)
  win_zero_kernel<<<e->n_sm * 8, 256, 0, st>>>(t.slots.as<uint32_t>(), t.win_state.as<uint32_t>(), nullptr, w0, (uint32_t)((t.local_size >> WIN_LG) - w0));
  JF_LAUNCHED();
  CUDA_OK(e, cudaGetLastError());
  t.materialized = t.local_size;
  return JFGPU_OK;
}

// The matrix large_hash::array draws for a table of 2^lsize slots (large_hash_array.hpp:992-1002)
jfb::gf2_matrix draw_matrix(jfgpu_engine* e, uint64_t requested_size, unsigned lsize) {
  const unsigned kbits = 2 * e->k;
  const bool smaller = kbits >= 64 || requested_size < ((uint64_t)1 << kbits);
  if(!smaller) return jfb::gf2_matrix::identity(kbits);
  jfb::gf2_matrix m(lsize, kbits);
  return m.randomize_pseudo_inverse(e->rng);
}

template<typename F>
int dispatch(jfgpu_engine* e, unsigned kw, unsigned sb, F&& f) {
  if(kw == 1 && sb == 32)  return f(std::integral_constant<int, 1>(), std::integral_constant<int, 32>());
  if(kw == 1 && sb == 64)  return f(std::integral_constant<int, 1>(), std::integral_constant<int, 64>());
  if(kw == 1 && sb == 128) return f(std::integral_constant<int, 1>(), std::integral_constant<int, 128>());
  if(kw == 2 && sb == 64)  return f(std::integral_constant<int, 2>(), std::integral_constant<int, 64>());
  if(kw == 2 && sb == 128) return f(std::integral_constant<int, 2>(), std::integral_constant<int, 128>());
  return fail(e, JFGPU_ERR_ARG, "unsupported key/slot combination");
}


// The kernels of four-word keys, compiled in jf_wide.cu (jf_wide.cuh), with their types
struct WideKernels {
  void (*extract_count)(const CountArgs, const PartDev);
  void (*extract_query)(const CountArgs, const PartDev);
  void (*insert_keys)(TableDev, const uint64_t*, uint32_t, const uint64_t*, const uint64_t*, uint64_t);
  void (*collect)(const CollectArgs);
  void (*dump_count)(const DumpArgs);
  void (*dump_emit)(const DumpArgs);
  void (*lookup)(TableDev, const uint64_t*, uint32_t, const uint64_t*, uint64_t, uint64_t*, uint32_t);
  void (*query_lookup)(TableDev, const uint64_t*, uint32_t, const uint64_t*, const uint32_t*, uint32_t, uint64_t, uint32_t, uint32_t,
                       uint64_t*, unsigned long long*);
  void (*query_decode)(const uint8_t*, uint64_t, uint32_t, uint32_t, uint64_t*, uint64_t*);
  void (*query_format)(const uint64_t*, const uint64_t*, const uint32_t*, uint32_t, uint64_t, uint64_t, const unsigned long long*,
                       uint32_t, uint8_t*);
  void (*histogram)(TableDev, uint64_t, unsigned long long*, uint32_t);
  void (*extract_route)(const CountArgs, const PartDev);
};
template<typename F> void wide_cast(F& f, const void* p) { f = reinterpret_cast<F>(const_cast<void*>(p)); }
const WideKernels& wide_kernels() {
  static const WideKernels w = [] {
    const jfw::Kernels& p = jfw::kernels();
    WideKernels k;
    wide_cast(k.extract_count, p.extract_count); wide_cast(k.extract_query, p.extract_query); wide_cast(k.insert_keys, p.insert_keys);
    wide_cast(k.collect, p.collect); wide_cast(k.dump_count, p.dump_count); wide_cast(k.dump_emit, p.dump_emit);
    wide_cast(k.lookup, p.lookup); wide_cast(k.query_lookup, p.query_lookup); wide_cast(k.query_decode, p.query_decode);
    wide_cast(k.query_format, p.query_format); wide_cast(k.histogram, p.histogram); wide_cast(k.extract_route, p.extract_route);
    return k;
  }();
  return w;
}
size_t wide_extract_smem(size_t lut_bytes) { return jfw::extract_smem(lut_bytes); }

// The kernels of sharded Bloom counting, compiled in jf_bloom.cu (jf_bloom.cuh), with their types
struct BloomKernels {
  void (*insert_keys[5])(TableDev, const uint64_t*, uint32_t, const uint64_t*, uint64_t, BloomDev);   // dispatch order
  void (*stage_keys[2])(TableDev, PartDev, const uint64_t*, uint32_t, const uint64_t*, uint64_t, BloomDev);
  void (*fold)(uint32_t*, const uint32_t*, uint64_t);
};
const BloomKernels& bloom_kernels() {
  static const BloomKernels b = [] {
    const jfbl::Kernels& p = jfbl::kernels();
    BloomKernels k;
    for(int i = 0; i < 5; ++i) wide_cast(k.insert_keys[i], p.insert_keys[i]);
    for(int i = 0; i < 2; ++i) wide_cast(k.stage_keys[i], p.stage_keys[i]);
    wide_cast(k.fold, p.fold);
    return k;
  }();
  return b;
}
// index of insert_keys_bf_kernel<KW, SB> in BloomKernels::insert_keys
template<int KW, int SB> constexpr int bloom_insert_index() { return KW == 1 ? (SB == 32 ? 0 : SB == 64 ? 1 : 2) : (SB == 64 ? 3 : 4); }

template<int NTH>
size_t count_smem_bytes(size_t lut_bytes, size_t stage_bytes, size_t bloom_bytes = 0, bool fast = false) {
  const size_t part = fast ? FAST_SMEM : (stage_bytes ? PMAX * 4 + stage_bytes : 0);
  return ((sizeof(ExtractSmemT<NTH>) + 15) & ~(size_t)15) + lut_bytes + part + bloom_bytes;
}

int ensure_scratch(jfgpu_engine* e, uint64_t n_tiles) {
  if(n_tiles <= e->scratch_tiles) return JFGPU_OK;
  uint64_t want = std::max<uint64_t>(n_tiles, 1024);
  CUDA_OK(e, cudaStreamSynchronize(e->cs));
  e->scratch_tiles = 0;
  CUDA_OK(e, make_all(need(e->nlA, want * 8), need(e->nlB, want * 8), need(e->cntA, want * 4), need(e->cntB, want * 4), need(e->tstate, want)));
  e->scratch_tiles = want;
  return JFGPU_OK;
}

// ---- partitioned insertion: geometry, pool, drain --------------------------------------
// the ring memory of the staging kernels (RING_P * RING records) shared out among P regions
uint32_t ring_len_for(uint32_t P) {
  uint32_t p2 = 1; while(p2 < P) p2 <<= 1;
  const uint32_t len = p2 >= RING_P ? RING : RING * (RING_P / p2);
  return std::min<uint32_t>(len, 1024);
}
PartDev part_dev(const jfgpu_engine* e) {
  PartDev d;
  memset(&d, 0, sizeof(d));
  const PartState& ps = e->part;
  d.P = ps.P; d.region_bits = ps.region_bits; d.rec_bytes = ps.rec_bytes; d.cap = ps.cap; d.flush_min = ps.flush_min;
  d.chunk_recs = CHUNK_BYTES / std::max(1u, ps.rec_bytes); d.n_chunks = ps.n_chunks; d.stage_bytes = ps.stage_bytes;
  d.margin = ps.margin;
  d.lazy_win = e->tab.materialized < e->tab.local_size ? e->tab.win_state.as<uint32_t>() : nullptr;
  d.arena_chunks = ps.arena_chunks;
  d.ring_len = ring_len_for(ps.P ? ps.P : 1);
  d.pool = ps.pool.as<uint8_t>(); d.pool_next = ps.pool_next.as<unsigned int>(); d.n_units = d.pool_next + ps.n_arenas; d.dir = ps.dir.as<uint2>();
  d.cta_chunk = ps.cta_chunk.as<uint32_t>(); d.cta_fill = ps.cta_fill.as<uint32_t>();
  d.spill_keys = ps.spill_keys.as<uint64_t>(); d.spill_counts = ps.spill_counts.as<uint64_t>();
  d.spill_n = ps.spill_n.as<unsigned long long>(); d.spill_cap = ps.spill_cap;
  return d;
}

// The send pool of sharded counting as K1 sees it: regions of the GLOBAL table, arenas by owning shard.
PartDev shard_send_dev(const jfgpu_engine* e, int bank) {
  PartDev d;
  memset(&d, 0, sizeof(d));
  const ShardState& sh = e->sh;
  const uint32_t G = e->p.n_shards;
  d.P = sh.P; d.region_bits = sh.sbits; d.rec_bytes = 4; d.chunk_recs = CHUNK_BYTES / 4;
  d.n_chunks = (uint32_t)(sh.arena_chunks * G); d.arena_chunks = (uint32_t)sh.arena_chunks;
  d.by_owner = 1; d.owner_shift = sh.owner_shift;
  d.ring_len = ring_len_for(sh.P);
  // a chunk is closed once it might not take the records of one more ring pass (4 k-mers per thread of K1)
  { const double mean = 4096.0 / sh.P; d.margin = std::max<uint32_t>(2 * RING, (uint32_t)(mean + 6.0 * sqrt(mean) + 8.0)); }
  d.pool = sh.send_pool + (size_t)bank * G * sh.arena_chunks * CHUNK_BYTES;
  d.dir = sh.send_dir + (size_t)bank * G * sh.arena_chunks;
  d.pool_next = sh.pool_next[bank].as<unsigned int>(); d.n_units = d.pool_next + G;
  d.cta_chunk = sh.cta_chunk.as<uint32_t>(); d.cta_fill = sh.cta_fill.as<uint32_t>();
  return d;
}

// Decide whether (and how) the current table is filled region by region.
void part_configure(jfgpu_engine* e) {
  PartState& ps = e->part;
  const Table& t = e->tab;
  ps.P = 0;
  if(e->kw == 4) return;           // four-word keys: direct insertion only (no region records for the wide form)
  if(e->p.no_partition || t.bytes() < ((size_t)(e->p.part_min_mb ? e->p.part_min_mb : 256) << 20)) return;       // small tables live in L2 anyway
  uint32_t P = 256;
  const size_t region_target = (size_t)(e->p.region_mb ? e->p.region_mb : 64) << 20;
  const size_t owned_bytes = (size_t)t.local_size * (t.slot_bits / 8);           // (without the overflow margin)
  while(P < (uint32_t)PMAX && (owned_bytes / P) > region_target) P <<= 1;
  // Smaller regions when that is what makes a record 4 bytes: the shared-memory window form of K2 (jf_window.cuh) takes only
  // 4-byte records of 32-bit slots, and is several times faster than the L2 form (2^33 slots at k=21: 64 MB regions need
  // 33-bit records, 32 MB regions 32-bit ones).  Only while K1 keeps its fast path (at most RING_P regions) and a region
  // still holds more than one window.
  if(t.slot_bits == 32 && t.local_lsize > ceil_log2(P)) {
    const uint32_t bits = t.local_lsize - ceil_log2(P) + t.hb, extra = bits > 32 ? bits - 32 : 0;
    if(extra && extra < 8 && (P << extra) <= (uint32_t)RING_P && t.local_lsize - ceil_log2(P << extra) > WIN_LG) P <<= extra;
  }
  for(;; P >>= 1) {
    if(P < 64 || t.local_lsize < 8 || (1u << (t.local_lsize - 8)) < P) return;
    const uint32_t region_bits = t.local_lsize - ceil_log2(P);
    const uint32_t bits = region_bits + t.hb;
    const uint32_t rec = bits <= 32 ? 4 : bits <= 64 ? 8 : bits <= 128 ? 16 : 0;
    // (a 16-byte record cannot hold hb + region_bits of a key field of 121..127 bits; those tables have at most 2^14
    // 128-bit slots, below the 1 MB floor of part_min_mb, so they never get here)
    if(!rec) return;
    // records arriving per region between two roll-over passes (one per window): 1024 threads x 32 symbols / P
    const double mean = 1024.0 * 32 / P;
    const uint32_t margin = (uint32_t)(mean + 6.0 * sqrt(mean) + 8.0);
    if(margin * 2 > CHUNK_BYTES / rec) return;               // chunks would be closed half empty: insert directly
    ps.P = P; ps.region_bits = region_bits; ps.rec_bytes = rec; ps.cap = 0; ps.flush_min = 0; ps.margin = margin;
    ps.stage_bytes = PMAX * 4;                               // the open-chunk ids (the counters are accounted separately)
    return;
  }
}

int part_alloc(jfgpu_engine* e) {
  PartState& ps = e->part;
  if(ps.pool.p) return JFGPU_OK;
  size_t free_b = 0, total_b = 0;
  CUDA_OK(e, cudaMemGetInfo(&free_b, &total_b));
  size_t want = e->p.pool_bytes ? (size_t)e->p.pool_bytes : std::min<size_t>((size_t)(free_b * 0.7), (size_t)64 << 30);
  const size_t floor_b = (size_t)e->n_sm * ps.P * CHUNK_BYTES * 2;        // every CTA keeps one open chunk per region
  if(want < floor_b) want = floor_b;
  // one arena per CTA of the staging kernels (persistent, one CTA per SM)
  ps.n_arenas = (uint32_t)e->n_sm;
  ps.arena_chunks = (uint32_t)std::min<size_t>(want / CHUNK_BYTES / ps.n_arenas, 0xFFFFFFF0u / ps.n_arenas);
  ps.n_chunks = ps.arena_chunks * ps.n_arenas;
  ps.spill_cap = (uint64_t)16 << 20;
  if(make_all(need(ps.pool, (size_t)ps.n_chunks * CHUNK_BYTES), need(ps.dir, (size_t)ps.n_chunks * 8), need(ps.order, (size_t)ps.n_chunks * 4),
              need(ps.pool_next, ((size_t)ps.n_arenas + 2) * 4), need(ps.cta_chunk, (size_t)e->n_sm * PMAX * 4),
              need(ps.cta_fill, (size_t)e->n_sm * PMAX * 4), need(ps.spill_keys, ps.spill_cap * 8 * e->kw), need(ps.spill_counts, ps.spill_cap * 8),
              need(ps.spill_n, 8), need(ps.hist, PMAX * 12), need(ps.start, PMAX * 4), need(ps.cursor, PMAX * 4), need(ps.unit_cursor, 8)) != cudaSuccess)
    return fail(e, JFGPU_ERR_NOMEM, "device allocation of the record pool failed");
  CUDA_OK(e, cudaMemsetAsync(ps.pool_next.p, 0, ps.pool_next.bytes, e->cs));
  CUDA_OK(e, cudaMemsetAsync(ps.spill_n.p, 0, 8, e->cs));
  CUDA_OK(e, cudaMemsetAsync(ps.cta_chunk.p, 0xFF, ps.cta_chunk.bytes, e->cs));
  CUDA_OK(e, cudaMemsetAsync(ps.cta_fill.p, 0, ps.cta_fill.bytes, e->cs));
  ps.bound_chunks = ps.P;
  ps.pending = false;
  CUDA_OK(e, cudaStreamSynchronize(e->cs));     // callers may continue on another stream
  return JFGPU_OK;
}

// records per region (chunk_hist_kernel), behind the chunk counts in `hist`
static unsigned long long* region_recs(PartState& ps) { return reinterpret_cast<unsigned long long*>(ps.hist.as<uint32_t>() + PMAX); }

int regrow(jfgpu_engine* e);
int spill_table(jfgpu_engine* e, uint64_t n_failed);
int read_stats(jfgpu_engine* e);
int bloom_draw(jfgpu_engine* e);
BloomDev bloom_dev(const jfgpu_engine* e);

// The failure counter of a drain, looked at one step late (hash_counter::add -> handle_full_ary) so that the device never
// waits for the host: two steps of failed keys fit the failure list (a step is at most fail_group records), and in a
// write-only drain so does the one deferred list that runs a step later still (fail_cap, jfgpu_create).
struct FailWatch {
  jfgpu_engine* e; cudaStream_t st;
  unsigned n = 0;                // copies posted since the drain began or the table was rebuilt
  // Post a copy of the live counter behind the work enqueued so far.  True when the copy of the step before shows failed
  // keys, or after the last step the copy just posted.
  bool step(bool last) {
    const int slot = (int)(n++ & 1);
    cudaMemcpyAsync(e->h_watch + slot, e->stats.as<unsigned long long>() + STAT_FAILED, 8, cudaMemcpyDeviceToHost, st);
    cudaEventRecord(e->ev_watch[slot], st);
    return (n > 1 && seen(slot ^ 1)) || (last && seen(slot));
  }
  bool seen(int slot) { cudaEventSynchronize(e->ev_watch[slot]); return e->h_watch[slot] != 0; }
};
static cudaError_t win_event(jfgpu_engine* e, cudaStream_t st) {
  if(e->wev_used == e->wev.size()) e->wev.emplace_back();
  Event& ev = e->wev[e->wev_used];
  if(!ev) { const cudaError_t c = make_all(need(ev, cudaEventDefault)); if(c != cudaSuccess) return c; }
  cudaEventRecord(ev, st);
  e->wev_used++;
  return cudaSuccess;
}
// Fold the event quadruples of the finished drain into win_ms (the stream must be idle).  Quadruple j belongs to the drain's
// j-th group with records: bucket pass + scan -> scatter; the exact pass -> hist when that group overflowed a bucket (w_flag[j]),
// else (a launch that returned at once) scatter; window insert -> insert.
static void resolve_win_events(jfgpu_engine* e, cudaStream_t st) {
  const size_t n_groups = e->wev_used / 4;
  std::vector<uint32_t> flag(n_groups);
  if(n_groups && (cudaMemcpyAsync(flag.data(), e->part.w_flag.p, n_groups * 4, cudaMemcpyDeviceToHost, st) != cudaSuccess ||
                  cudaStreamSynchronize(st) != cudaSuccess)) cudaGetLastError();
  for(size_t j = 0; j < n_groups; ++j)
    for(int q = 0; q < 3; ++q) {
      float ms = 0;
      const int to = q == 0 ? 1 : q == 1 ? (flag[j] ? 0 : 1) : 2;
      if(cudaEventElapsedTime(&ms, e->wev[4 * j + q], e->wev[4 * j + q + 1]) == cudaSuccess) e->win_ms[to] += ms; else cudaGetLastError();
    }
  e->wev_used = 0;
}
// k2_mode 3 and 4 take the window form too (include/jfgpu.h)
static bool window_enabled(jfgpu_engine* e, const PartDev& pd) {
  return (e->p.k2_mode == 0 || e->p.k2_mode == 3 || e->p.k2_mode == 4) && e->op == 0 && e->tab.slot_bits == 32 && pd.rec_bytes == 4 &&
         pd.region_bits > WIN_LG && pd.region_bits - WIN_LG <= 11;
}
// Whether a cleared table may stay zero in meaning only until its first drain: that drain takes the window form (plain
// insertion, no Bloom prefilter) and then writes every slot of [0, local_size), and a deferred probe reaches less than one
// region past its window.
static bool lazy_zero_ok(jfgpu_engine* e) {
  return e->part.P && e->bloom.mode == BLOOM_NONE && window_enabled(e, part_dev(e)) &&
         tri(e->tab.max_reprobe) < ((uint64_t)1 << e->part.region_bits);
}
// Insert everything that sits in the record pool (K1b), then the spill list.  One loop over the units (chunks in region
// order); a step is a group of regions in the window form of K2 (jf_window.cuh), a range of units in the L2 form, or, once
// the table has been doubled, a range in the rehash form.  With regrow enabled the steps are small enough for the failure
// list, and the failure counter is watched after each one.
int part_drain(jfgpu_engine* e, cudaStream_t st) {
  PartState& ps = e->part;
  if(!ps.P || !ps.pool.p || !ps.pending) return JFGPU_OK;
  PartDev pd = part_dev(e);
  // The form is decided once, for the geometry the records were written with.  A doubling in the middle of the drain does
  // not change it: it only narrows the key field (hb falls by one, the carried reprobe limit stays), so a 32-bit slot
  // stays 32-bit.
  const bool win = window_enabled(e, pd);
  const int g = e->n_sm * 4;
  if(!e->ev_d0) CUDA_OK(e, make_all(need(e->ev_d0, cudaEventDefault), need(e->ev_d1, cudaEventDefault)));
  cudaEventRecord(e->ev_d0, st);
  close_chunks_kernel<<<g, 256, 0, st>>>(pd, (uint32_t)e->n_sm); JF_LAUNCHED();
  CUDA_OK(e, cudaMemsetAsync(ps.hist.p, 0, PMAX * 12, st));
  chunk_hist_kernel<<<g, 256, 0, st>>>(pd, ps.hist.as<uint32_t>(), win ? region_recs(ps) : nullptr); JF_LAUNCHED();
  chunk_scan_kernel<<<1, 1024, 0, st>>>(pd.P, ps.hist.as<uint32_t>(), ps.start.as<uint32_t>(), ps.cursor.as<uint32_t>(), pd.n_units); JF_LAUNCHED();
  chunk_scatter_kernel<<<g, 256, 0, st>>>(pd, ps.cursor.as<uint32_t>(), ps.order.as<uint32_t>()); JF_LAUNCHED();
  CUDA_OK(e, cudaMemsetAsync(ps.unit_cursor.p, 0, 8, st));
  // geometry the records were written with (a regrow in the middle changes e->tab)
  const TableDev T0 = table_dev(e, e->tab);
  const bool careful = e->p.allow_regrow != 0 || e->spill_fn != nullptr;
  unsigned int n_units = 0xFFFFFFFFu;           // (not read when one range of the L2 form takes them all)
  if(careful || win) {
    CUDA_OK(e, cudaMemcpyAsync(&n_units, pd.n_units, 4, cudaMemcpyDeviceToHost, st));
    CUDA_OK(e, cudaStreamSynchronize(st));
    n_units = std::min(n_units, ps.n_chunks);
  }
  const unsigned group = careful ? (unsigned)std::max<uint64_t>(1, e->fail_group / pd.chunk_recs) : 0xFFFFFFFFu;

  // window form: the first unit and the records of every region (chunk_scan_kernel, chunk_hist_kernel), on the host
  const uint32_t wpr_lg = win ? pd.region_bits - WIN_LG : 0;
  const uint64_t wpr = (uint64_t)1 << wpr_lg;
  const size_t scatter_smem = win_scatter_smem(WIN_ST_UNITS, WIN_ST_NBUF, (uint32_t)wpr);
  std::vector<uint32_t> start(pd.P + 1);
  std::vector<unsigned long long> recs(pd.P);
  auto win_begin = [&]() -> int {
    if(!ps.w_rec.p) {
      ps.w_rec_cap = (uint64_t)64 << 20;                       // records per group (256 MB)
      ps.w_def_cap = WIN_DEF_CAP;
      if(make_all(need(ps.w_rec, ps.w_rec_cap * 4 + 64), need(ps.w_start, (((size_t)WIN_MAX_G << 11) + 1) * 4), need(ps.w_cursor, ((size_t)WIN_MAX_G << 11) * 4),
                  need(ps.w_cnt, ((size_t)WIN_MAX_G << 11) * 4), need(ps.w_def_n, 16), need(ps.w_flag, PMAX * 4),
                  need(ps.w_def_pos[0], ps.w_def_cap * 8), need(ps.w_def_high[0], ps.w_def_cap * 4),
                  need(ps.w_def_pos[1], ps.w_def_cap * 8), need(ps.w_def_high[1], ps.w_def_cap * 4)) != cudaSuccess)
        return fail(e, JFGPU_ERR_NOMEM, "device allocation of the window buffers failed");
      CUDA_OK(e, cudaMemsetAsync(ps.w_def_n.p, 0, 16, st));
    }
    // the groups' overflow flags (k2_mode 3: set from the start, so that every group takes the exact placement)
    CUDA_OK(e, cudaMemsetAsync(ps.w_flag.p, e->p.k2_mode == 3 ? 1 : 0, PMAX * 4, st));
    CUDA_OK(e, cudaMemcpyAsync(start.data(), ps.start.p, (size_t)pd.P * 4, cudaMemcpyDeviceToHost, st));
    CUDA_OK(e, cudaMemcpyAsync(recs.data(), region_recs(ps), (size_t)pd.P * 8, cudaMemcpyDeviceToHost, st));
    CUDA_OK(e, cudaStreamSynchronize(st));
    start[pd.P] = n_units;
    for(uint32_t r = 0; r < pd.P; ++r) start[r] = std::min(start[r], n_units);
    cudaFuncSetAttribute(win_scatter_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)scatter_smem);
    cudaFuncSetAttribute(win_scatter_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)scatter_smem);
    return JFGPU_OK;
  };
  int rc = win ? win_begin() : JFGPU_OK;
  // Bucket capacity of a group: m = the largest mean of records per window over its regions.  A window's count is about
  // Poisson(m) for hashed input; m + 6 sqrt(m) + 16 leaves a window of iid input a chance of order 1e-9 to overflow, i.e.
  // a fallback to the exact placement about once in two thousand steps of configs[1] (half a million windows).  k2_mode 4
  // leaves no slack, so nearly every group overflows.  Regions join a group while its buckets fit the group buffer, and
  // so does its exact layout: the group's records (at most m per window on average) plus up to 3 padding records per
  // window, since every run starts on a 16-byte boundary.
  auto bucket_cap = [&](uint64_t m) -> uint64_t {
    const uint64_t c = e->p.k2_mode == 4 ? m : m + (uint64_t)std::ceil(6.0 * std::sqrt((double)m)) + 16;
    return (c + 3) & ~(uint64_t)3;
  };
  // Write-only drain (the table was zeroed lazily; only the windows K1 inserted into are in memory): win_insert2 loads no
  // other window, win_zero writes the other windows that get no record, and `materialized` follows group by group.  The
  // deferred records of a group are applied after the next group's windows are written (win_insert2 would overwrite what
  // they put there), the last group's once the rest of the table is zeroed.  Deferred list of group i: i & 1.
  bool zero = win && e->tab.materialized == 0;
  int def_wait = -1;                                         // deferred list not applied yet
  auto run_deferred = [&](int set) {
    WinDev wd;
    memset(&wd, 0, sizeof(wd));
    wd.def_pos = ps.w_def_pos[set].as<uint64_t>(); wd.def_high = ps.w_def_high[set].as<uint32_t>();
    wd.def_n = ps.w_def_n.as<unsigned long long>() + set; wd.def_cap = ps.w_def_cap;
    if(e->kw == 1) win_deferred_kernel<1><<<e->n_sm * 2, 256, 0, st>>>(T0, wd, e->tab.inv_lut.as<uint64_t>(), e->nbytes);
    else           win_deferred_kernel<2><<<e->n_sm * 2, 256, 0, st>>>(T0, wd, e->tab.inv_lut.as<uint64_t>(), e->nbytes);
    JF_LAUNCHED();
    cudaMemsetAsync(wd.def_n, 0, 8, st);
  };
  // the whole table in memory and every deferred record applied: the L2 and rehash forms, the collection of the old table
  // and the spill list read the slots
  auto end_zero = [&]() -> int {
    const int rc2 = table_materialize(e, e->tab, st);
    if(rc2 || !zero) return rc2;
    if(def_wait >= 0) run_deferred(def_wait);
    def_wait = -1; zero = false;
    return JFGPU_OK;
  };
  DevBuf old_inv;     // inverse tables of the geometry the records belong to, once the table has been rebuilt
  bool rebuilt = false;
  // units [done, upto) in the L2 form, or in the rehash form once the table has been rebuilt
  auto range = [&](unsigned done, unsigned upto) -> int {
    int rc2 = end_zero();
    if(rc2) return rc2;
    cudaMemsetAsync(ps.unit_cursor.p, 0, 8, st);
    const TableDev T = table_dev(e, e->tab);
    if(rebuilt) {
      const size_t smem = (size_t)e->nbytes * 256 * 8 * 2;
      rc2 = dispatch(e, e->kw, e->tab.slot_bits, [&](auto KW, auto SB) -> int {
        auto kern = rehash_chunks_kernel<decltype(KW)::value, decltype(SB)::value>;
        cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        kern<<<e->n_sm, 512, smem, st>>>(T, T0, pd, ps.order.as<uint32_t>(), ps.unit_cursor.as<unsigned int>(), done, upto,
                                        old_inv.as<uint64_t>(), e->tab.lut.as<uint64_t>(), e->nbytes);
        return JFGPU_OK;
      });
    } else if(e->op == 0 && e->tab.slot_bits == 32 && pd.rec_bytes == 4 && e->p.k2_mode != 2) {
      // lean 32-bit specialisation: 2 CTAs x 1024 threads per SM
      if(e->kw == 1) insert_chunks32_kernel<1><<<e->n_sm * 2, 768, 0, st>>>(T, pd, ps.order.as<uint32_t>(), ps.unit_cursor.as<unsigned int>(), done, upto, e->tab.inv_lut.as<uint64_t>(), e->nbytes);
      else           insert_chunks32_kernel<2><<<e->n_sm * 2, 768, 0, st>>>(T, pd, ps.order.as<uint32_t>(), ps.unit_cursor.as<unsigned int>(), done, upto, e->tab.inv_lut.as<uint64_t>(), e->nbytes);
    } else
      rc2 = dispatch(e, e->kw, e->tab.slot_bits, [&](auto KW, auto SB) -> int {
        insert_chunks_kernel<decltype(KW)::value, decltype(SB)::value><<<e->n_sm * 2, 512, 0, st>>>(
            T, pd, ps.order.as<uint32_t>(), ps.unit_cursor.as<unsigned int>(), done, upto, e->tab.inv_lut.as<uint64_t>(), e->nbytes);
        return JFGPU_OK;
      });
    if(!rc2) JF_LAUNCHED();
    return rc2;
  };

  FailWatch watch{e, st};
  unsigned done = 0;
  uint32_t r0 = 0, ng = 0;       // window form: the first region of the next group, the groups so far
  bool ranged = false;           // a range of the L2 or rehash form has run (they run at least one, an empty one too)
  while(!rc) {
    const bool window = win && !rebuilt;
    if(done >= n_units && (window || ranged)) break;
    unsigned upto = 0;
    if(!window) {
      upto = (unsigned)std::min<uint64_t>((uint64_t)done + group, n_units);
      rc = range(done, upto);
      ranged = true;
    } else {
      WinDev wd;
      memset(&wd, 0, sizeof(wd));
      uint32_t G = 0, stiles = 0;
      uint64_t m = 0, cap = 0;
      while(r0 + G < pd.P && G < WIN_MAX_G) {
        const uint32_t nu = start[r0 + G + 1] - start[r0 + G];
        if(careful && start[r0 + G + 1] - start[r0] > group) break;
        const uint64_t m2 = std::max<uint64_t>(m, (recs[r0 + G] + wpr - 1) / wpr), cap2 = bucket_cap(m2);
        if((G + 1) * wpr * std::max(cap2, m2 + 3) > ps.w_rec_cap) break;
        m = m2; cap = cap2;
        wd.stile_first[G] = stiles; wd.unit_first[G] = start[r0 + G];
        stiles += (nu + WIN_ST_UNITS - 1) / WIN_ST_UNITS;
        ++G;
      }
      if(G == 0) {
        // a single region holds more records than the group buffer (heavily repeated k-mers): the L2 form for it, whose
        // probes read the slots of the next region too
        upto = start[r0 + 1]; r0 += 1;
        rc = range(done, upto);
      } else {
        wd.stile_first[G] = stiles; wd.unit_first[G] = start[r0 + G];
        wd.g0 = r0; wd.G = G; wd.wpr_lg = wpr_lg; wd.n_tiles = stiles; wd.cap = (uint32_t)cap;
        wd.overflow = ps.w_flag.as<uint32_t>() + e->wev_used / 4;      // (flag j: the drain's j-th group with records, resolve_win_events)
        wd.wstart = ps.w_start.as<uint32_t>(); wd.wcursor = ps.w_cursor.as<uint32_t>(); wd.wcnt = ps.w_cnt.as<uint32_t>();
        wd.wrec = ps.w_rec.as<uint32_t>(); wd.wrec_cap = ps.w_rec_cap;
        const int set = zero ? (int)(ng & 1) : 0;
        wd.def_pos = ps.w_def_pos[set].as<uint64_t>(); wd.def_high = ps.w_def_high[set].as<uint32_t>();
        wd.def_n = ps.w_def_n.as<unsigned long long>() + set; wd.def_cap = ps.w_def_cap;
        wd.lazy_win = zero ? e->tab.win_state.as<uint32_t>() : nullptr;
        const uint32_t hb = e->tab.fbits - e->tab.rbits;
        // the deferred records, once every slot they can reach holds its value in memory
        auto settle = [&]() {
          if(!zero) { if(stiles) run_deferred(set); return; }
          e->tab.materialized = (uint64_t)(r0 + G) << pd.region_bits;
          if(def_wait >= 0) run_deferred(def_wait);
          def_wait = stiles ? set : -1;
        };
        ++ng;
        if(stiles) {
          CUDA_OK(e, cudaMemsetAsync(ps.w_cursor.p, 0, ((size_t)G << wpr_lg) * 4, st));
          CUDA_OK(e, win_event(e, st));
          win_scatter_kernel<true><<<std::min<uint32_t>(stiles, e->n_sm), WIN_ST_NTH, scatter_smem, st>>>(pd, wd, ps.order.as<uint32_t>(), hb); JF_LAUNCHED();
          win_scan_kernel<<<1, 1024, 0, st>>>(wd, T0.stats); JF_LAUNCHED();
          CUDA_OK(e, win_event(e, st));
          win_scatter_kernel<false><<<std::min<uint32_t>(stiles, e->n_sm), WIN_ST_NTH, scatter_smem, st>>>(pd, wd, ps.order.as<uint32_t>(), hb);
          JF_LAUNCHED();
          CUDA_OK(e, win_event(e, st));
          if(e->kw == 1) {
            cudaFuncSetAttribute(win_insert2_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)WIN2_SMEM);
            win_insert2_kernel<1><<<e->n_sm, WIN2_NTH, WIN2_SMEM, st>>>(T0, pd, wd, e->tab.inv_lut.as<uint64_t>(), e->nbytes); JF_LAUNCHED();
          } else {
            cudaFuncSetAttribute(win_insert2_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)WIN2_SMEM);
            win_insert2_kernel<2><<<e->n_sm, WIN2_NTH, WIN2_SMEM, st>>>(T0, pd, wd, e->tab.inv_lut.as<uint64_t>(), e->nbytes); JF_LAUNCHED();
          }
          if(zero) {
            win_zero_kernel<<<e->n_sm * 4, 256, 0, st>>>(e->tab.slots.as<uint32_t>(), wd.lazy_win, wd.wcnt, (uint64_t)r0 << wpr_lg, G << wpr_lg);
            JF_LAUNCHED();
          }
          settle();
          CUDA_OK(e, win_event(e, st));
        } else {
          if(zero) {
            win_zero_kernel<<<e->n_sm * 4, 256, 0, st>>>(e->tab.slots.as<uint32_t>(), wd.lazy_win, nullptr, (uint64_t)r0 << wpr_lg, G << wpr_lg);
            JF_LAUNCHED();
          }
          settle();
        }
        upto = start[r0 + G]; r0 += G;
      }
    }
    if(rc) break;
    done = upto;
    if(!careful) continue;
    const bool last = done >= n_units;
    if(last) { rc = end_zero(); if(rc) break; }      // (the last deferred records may fail too: the last copy follows them)
    if(!watch.step(last)) continue;
    // keys found no slot: the old table is collected next, all of it in memory with every deferred record applied; a copy
    // of the inverse tables the pending records were written against is kept, the rest goes through the rehash form
    rc = end_zero();
    if(rc) break;
    cudaStreamSynchronize(st);
    watch.n = 0;                 // the steps launched so far are complete: start the look-behind afresh
    if(!rebuilt) {
      if(old_inv.alloc(e->tab.inv_lut.bytes) != cudaSuccess) { cudaGetLastError(); rc = fail(e, JFGPU_ERR_NOMEM, "device allocation failed"); break; }
      cudaMemcpyAsync(old_inv.p, e->tab.inv_lut.p, e->tab.inv_lut.bytes, cudaMemcpyDeviceToDevice, e->cs);
      cudaStreamSynchronize(e->cs);
      rebuilt = true;
    }
    rc = regrow(e);
  }
  if(!rc) rc = end_zero();
  if(!rc) {
    // the spilled keys carry full keys: plain insertion into whatever the table is now
    TableDev T = table_dev(e, e->tab);
    const size_t smem = (size_t)e->nbytes * 256 * 8;
    rc = dispatch(e, e->kw, e->tab.slot_bits, [&](auto KW, auto SB) -> int {
      auto kern = insert_spill_kernel<decltype(KW)::value, decltype(SB)::value>;
      cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
      kern<<<e->n_sm * 2, 256, smem, st>>>(T, e->tab.lut.as<uint64_t>(), e->nbytes, pd);
      return JFGPU_OK;
    });
    if(!rc) JF_LAUNCHED();
  }
  cudaMemsetAsync(ps.pool_next.p, 0, ps.pool_next.bytes, st);
  cudaMemsetAsync(ps.spill_n.p, 0, 8, st);
  cudaEventRecord(e->ev_d1, st);
  cudaStreamSynchronize(st);
  { float ms = 0; if(cudaEventElapsedTime(&ms, e->ev_d0, e->ev_d1) == cudaSuccess) e->drain_ms += ms; else cudaGetLastError(); }
  resolve_win_events(e, st);
  ps.pending = false;
  if(rebuilt) {                  // (old_inv goes when the drain returns; the stream is idle)
    part_configure(e);
    if(!ps.P) ps = PartState();  // a table no longer filled region by region gives its record pool back
  }
  ps.bound_chunks = ps.P;
  if(rc) return rc;
  CUDA_OK(e, cudaGetLastError());
  return JFGPU_OK;
}

// records a closed chunk of the pool holds at least
uint64_t chunk_usable(const PartState& ps) { return CHUNK_BYTES / ps.rec_bytes - ps.margin; }
// chunks of one arena that `per_cta` records may take: the ones they fill, plus those the roll-over passes may leave nearly
// empty
uint64_t chunks_for(const PartState& ps, uint64_t per_cta) { return per_cta / chunk_usable(ps) + 2; }

// Reserve `need` chunks of every arena for one launch that writes records into the pool (ps.bound_chunks is a host-side
// upper bound of the chunks in use in any one arena); drain first when the bound says an arena could fill up.  When that
// drain doubled the table and the new one is not filled region by region (ps.P == 0), nothing is reserved: the caller
// inserts directly.
int part_reserve(jfgpu_engine* e, cudaStream_t st, uint64_t need, const char* too_small) {
  PartState& ps = e->part;
  if(ps.bound_chunks + need > ps.arena_chunks) {
    const int rc = part_drain(e, st);
    if(rc || !ps.P) return rc;
  }
  if(ps.bound_chunks + need > ps.arena_chunks) return fail(e, JFGPU_ERR_NOMEM, too_small);
  ps.bound_chunks += need;
  ps.pending = true;
  return JFGPU_OK;
}

// no more text per launch than an empty arena can take (small pools: tests, tables that leave little memory)
size_t part_cap_len(const jfgpu_engine* e, size_t len) {
  const PartState& ps = e->part;
  if(!ps.P || !ps.arena_chunks) return len;
  const uint64_t room = ps.arena_chunks > ps.P + 8 ? ps.arena_chunks - ps.P - 8 : 1;
  const uint64_t tiles_per_cta = std::max<uint64_t>(room * chunk_usable(ps) / (1024 * 32), 1);
  const uint64_t cap = tiles_per_cta * (1024 * 32 - HALO) * (uint64_t)e->n_sm / 2;
  return len > cap ? (size_t)std::max<uint64_t>(cap & ~(uint64_t)15, 16) : len;
}

// the quality threshold in force: the PRIME pass of --if reads its files without it (count_main.cc:289-295 uses mer_counter there)
// (a query reads its text as query_from_sequence does, without qualities)
static uint32_t eff_min_qual(const jfgpu_engine* e) { return e->op == JFGPU_OP_PRIME || e->querying ? 0u : e->p.min_qual; }

// What K1 does with a batch (the values are what CountArgs.mode carries)
enum K1Use : uint32_t {
  K1_COUNT = 0,      // count: into the table, or as region records into the pool
  K1_ROUTE = 1,      // keys into the caller's buckets by owning shard
  K1_SEND = 2,       // region records of the GLOBAL table into a bank of the record exchange's send pool
  K1_QUERY = 4,      // the keys of a query, in input order, into the buffers e->qb[e->q_cur]
};

// One batch of device-resident text through K0a, K0b, K1 on `stream`.
int run_batch(jfgpu_engine* e, const uint8_t* dev, uint64_t n, uint64_t n_look, cudaStream_t stream, K1Use use, uint64_t n_back = 0,
              int bank = 0, uint64_t* route_keys = nullptr, unsigned long long* route_counts = nullptr, uint64_t route_cap = 0) {
  if(n == 0) return JFGPU_OK;
  PartState& ps = e->part;
  const bool bc_build = e->bloom.mode == BLOOM_COUNT;
  bool part = use == K1_COUNT && ps.P != 0 && !bc_build;
  int rc;
  if(e->bloom.mode != BLOOM_NONE && !e->bloom.drawn && (e->op != JFGPU_OP_PRIME || bc_build)) { rc = bloom_draw(e); if(rc) return rc; }
  if(part) {
    rc = part_alloc(e);
    if(rc) return rc;
    // a CTA sees ceil(tiles / CTAs) tiles, one record per input byte at most
    const uint64_t tile_b = 1024 * 32 - HALO;
    const uint64_t tiles = (n + tile_b - 1) / tile_b;
    rc = part_reserve(e, stream, chunks_for(ps, (tiles + e->n_sm - 1) / e->n_sm * tile_b), "record pool smaller than one batch");
    if(rc) return rc;
    part = ps.P != 0;
  }
  if(!part && use == K1_COUNT && !bc_build) {            // K1 inserts into the table itself
    rc = table_materialize(e, e->tab, stream);
    if(rc) return rc;
  }
  const bool shard_send = use == K1_SEND;
  const bool query = use == K1_QUERY;
  const uint32_t tile = (part || shard_send ? 1024 : 512) * 32 - HALO;
  const uint64_t n_tiles = (n + tile - 1) / tile;
  rc = ensure_scratch(e, n_tiles);
  if(rc) return rc;
  const int g0 = (int)std::min<uint64_t>(n_tiles, (uint64_t)e->n_sm * 8);
  nl_scan_kernel<<<g0, 256, 0, stream>>>(dev, n, n_tiles, tile, e->nlA.as<long long>(), e->nlB.as<long long>(), e->cntA.as<uint32_t>(), e->cntB.as<uint32_t>());
  JF_LAUNCHED();
  if(e->format == 1)
    tile_state_fastq_kernel<<<1, 1024, 0, stream>>>(n_tiles, e->cntA.as<uint32_t>(), e->cntB.as<uint32_t>(), e->carry[e->carry_cur].as<Carry>(), e->tstate.as<uint8_t>());
  else
    tile_state_kernel<<<1, 1024, 0, stream>>>(dev, n_tiles, tile, e->nlA.as<long long>(), e->nlB.as<long long>(),
                                              e->carry[e->carry_cur].as<Carry>(), e->tstate.as<uint8_t>(), eff_min_qual(e));
  JF_LAUNCHED();
  CountArgs a;
  memset(&a, 0, sizeof(a));
  a.in = dev; a.n = n; a.n_look = n_look; a.n_tiles = n_tiles;
  a.tile_state = e->tstate.as<uint8_t>();
  a.carry_in = e->carry[e->carry_cur].as<Carry>();
  a.carry_out = e->carry[e->carry_cur ^ 1].as<Carry>();
  a.lut = e->tab.hash_fast ? e->tab.lut11.as<uint64_t>() : e->tab.lut.as<uint64_t>();
  a.hash_fast = e->tab.hash_fast ? 1 : 0; a.n_prow = e->tab.n_prow;
  a.lut_bytes = e->tab.hash_fast ? 4 * 2048 * 4 : e->nbytes * 256 * 8;
  for(unsigned i = 0; i < 8; ++i) a.prow[i] = e->tab.prow[i];
  a.min_qual = eff_min_qual(e); a.n_back = n_back;
  a.k = e->k; a.canonical = e->p.canonical; a.nbytes = e->nbytes; a.mode = use; a.format = (uint32_t)e->format;
  a.T = table_dev(e, e->tab);
  a.bloom = bloom_dev(e);
  // a shard's --bf-size prefilter sees every occurrence of its keys only on the owner (jfgpu_insert_keys): the sender
  // routes them unfiltered.  (A loaded counter, --bc, is a fixed read-only test: the sender applies it.)
  if(use == K1_ROUTE && a.bloom.mode == BLOOM_FILTER) memset(&a.bloom, 0, sizeof(a.bloom));
  const size_t bloom_smem = a.bloom.mode ? (size_t)e->nbytes * 256 * 8 * 2 : 0;
  if(bc_build) { a.lut = nullptr; a.lut_bytes = 0; a.hash_fast = 0; }
  a.route_keys = route_keys; a.route_counts = route_counts; a.route_cap = route_cap; a.shard_bits = e->shard_bits;
  if(query) {                                   // no hash, no filter: the keys themselves, in input order
    a.lut = nullptr; a.lut_bytes = 0; a.hash_fast = 0; memset(&a.bloom, 0, sizeof(a.bloom));
    a.q_keys = (e->seaming ? e->seam_keys : e->qb[e->q_cur].keys).as<uint64_t>();
    a.q_cnt = (e->seaming ? e->seam_cnt : e->qb[e->q_cur].cnt).as<uint32_t>(); a.q_tile_cap = tile;
  }
  PartDev pd = shard_send ? shard_send_dev(e, bank) : part_dev(e);
  auto launch = [&](auto kern, int nth, size_t smem, bool one_per_sm) -> int {
    cudaError_t c = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if(c != cudaSuccess) return fail(e, JFGPU_ERR_CUDA, std::string("cudaFuncSetAttribute: ") + cudaGetErrorString(c));
    cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
    // persistent CTAs: exactly as many as are resident at once (a multiple of the SM count)
    int per_sm = 1;
    if(!one_per_sm && (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, nth, smem) != cudaSuccess || per_sm < 1)) { cudaGetLastError(); per_sm = 1; }
    // (sharded counting leaves a few SMs to the collective that runs beside K1)
    const int sms = shard_send && e->n_sm > 32 ? e->n_sm - (int)SHARD_RESERVED_SMS : e->n_sm;
    const int grid = (int)std::min<uint64_t>(n_tiles, (uint64_t)sms * per_sm);
    if(query) { kern<<<grid, nth, smem, stream>>>(a, pd); return JFGPU_OK; }     // (the counting statistics leave a query out)
    if(e->kev_used == e->kev.size()) e->kev.resize(e->kev_used + 2);
    if(!e->kev[e->kev_used]) {
      c = make_all(need(e->kev[e->kev_used], cudaEventDefault), need(e->kev[e->kev_used + 1], cudaEventDefault));
      if(c != cudaSuccess) return fail(e, JFGPU_ERR_CUDA, std::string("cudaEventCreate: ") + cudaGetErrorString(c));
    }
    cudaEventRecord(e->kev[e->kev_used], stream);
    kern<<<grid, nth, smem, stream>>>(a, pd);
    cudaEventRecord(e->kev[e->kev_used + 1], stream);
    e->kev_used += 2;
    return JFGPU_OK;
  };
  // four-word keys (jf_wide.cu): direct insertion (MODE 0), keys bucketed by owner (MODE 1) or query extraction (MODE 3)
  if(e->kw == 4) {
    if(query) rc = launch(wide_kernels().extract_query, 512, wide_extract_smem(0), false);
    else if(part || shard_send || a.bloom.mode) rc = fail(e, JFGPU_ERR_ARG, "k > 64 takes neither region records, the record exchange nor a Bloom filter");
    else if(use == K1_ROUTE) rc = launch(wide_kernels().extract_route, 512, wide_extract_smem(a.lut_bytes), false);
    else rc = launch(wide_kernels().extract_count, 512, wide_extract_smem(a.lut_bytes), false);
  } else rc = dispatch(e, e->kw, e->tab.slot_bits, [&](auto KW, auto SB) -> int {
    constexpr int kw = decltype(KW)::value, sb = decltype(SB)::value;
    if(shard_send) {
      if(kw == 1 && e->tab.n_prow <= 2) return launch(extract_kernel<1, sb, 2, 1024, true, 2>, 1024, count_smem_bytes<1024>(a.lut_bytes, 0, 0, true), true);
      if(kw == 1) return launch(extract_kernel<1, sb, 2, 1024, true, 6>, 1024, count_smem_bytes<1024>(a.lut_bytes, 0, 0, true), true);
      return fail(e, JFGPU_ERR_STATE, "internal: record exchange with a two-word key");
    }
    if(part) {
      // the all-32-bit tail: 11-bit-table hash with at most two parity rows, 4-byte records, one shard, region index and
      // record fields inside 32 bits
      const bool fast = kw == 1 && e->tab.hash_fast && e->tab.n_prow <= 6 && ps.rec_bytes == 4 && e->shard_bits == 0 &&
                        ps.region_bits >= 2 && ps.region_bits < 32 && e->tab.lsize <= 38 && e->tab.lsize >= ps.region_bits &&
                        ps.P <= RING_P && !a.bloom.mode;
      if(kw == 1 && fast && e->tab.n_prow <= 2) return launch(extract_kernel<1, sb, 2, 1024, true, 2>, 1024, count_smem_bytes<1024>(a.lut_bytes, ps.stage_bytes, 0, true), true);
      if(kw == 1 && fast) return launch(extract_kernel<1, sb, 2, 1024, true, 6>, 1024, count_smem_bytes<1024>(a.lut_bytes, ps.stage_bytes, 0, true), true);
      return launch(extract_kernel<kw, sb, 2, 1024, false>, 1024, count_smem_bytes<1024>(a.lut_bytes, ps.stage_bytes, bloom_smem), true);
    }
    if(query) return launch(extract_kernel<kw, 64, 3, 512, false>, 512, count_smem_bytes<512>(0, 0, 0), false);
    if(use == K1_ROUTE) return launch(extract_kernel<kw, sb, 1, 512, false>, 512, count_smem_bytes<512>(a.lut_bytes, 0, bloom_smem), false);
    return launch(extract_kernel<kw, sb, 0, 512, false>, 512, count_smem_bytes<512>(a.lut_bytes, 0, bloom_smem), false);
  });
  if(rc) return rc;
  JF_LAUNCHED();
  CUDA_OK(e, cudaGetLastError());
  e->carry_cur ^= 1;
  return JFGPU_OK;
}

// ---- Bloom filter / counter ------------------------------------------------------------
// bloom_base::opt_m / opt_k (bloom_common.hpp:62-67)
int bloom_setup(jfgpu_engine* e, uint32_t mode, uint64_t n, double fp) {
  BloomState& b = e->bloom;
  if(fp <= 0.0) fp = mode == BLOOM_COUNT ? 0.001 : 0.01;          // bc_main_cmdline.yaggo / count_main_cmdline.yaggo defaults
  if(fp >= 1.0) return fail(e, JFGPU_ERR_ARG, "false positive rate must be in (0, 1)");
  const double LOG2 = 0.6931471805599453, LOG2_SQ = 0.4804530139182014;
  b.m = n * (uint64_t)lrint(-log(fp) / LOG2_SQ);
  b.k = (uint32_t)lrint(-log(fp) / LOG2);
  if(b.m == 0 || b.k == 0) return fail(e, JFGPU_ERR_ARG, "empty Bloom filter (size and false positive rate give no bits)");
  b.mode = mode;
  b.inv = b.m == 1 ? ~(uint64_t)0 : (uint64_t)(((unsigned __int128)1 << 64) / b.m);
  b.n_words = mode == BLOOM_COUNT ? (b.m + 15) / 16 : (b.m + 31) / 32;
  if(b.bits.alloc((size_t)b.n_words * 4 + 16) != cudaSuccess) { cudaGetLastError(); return fail(e, JFGPU_ERR_NOMEM, "Failed to allocate the Bloom filter in device memory"); }
  CUDA_OK(e, cudaMemsetAsync(b.bits.p, 0, b.bits.bytes, e->cs));
  if(mode == BLOOM_FILTER) {
    CUDA_OK(e, b.locks.alloc((size_t)4 << 20));
    CUDA_OK(e, cudaMemsetAsync(b.locks.p, 0, b.locks.bytes, e->cs));
  }
  b.drawn = false;
  return JFGPU_OK;
}
int bloom_upload_matrices(jfgpu_engine* e) {
  BloomState& b = e->bloom;
  std::vector<uint64_t> l1 = build_lut(b.M1, e->nbytes), l2 = build_lut(b.M2, e->nbytes);
  CUDA_OK(e, b.lut1.alloc(l1.size() * 8));
  CUDA_OK(e, b.lut2.alloc(l2.size() * 8));
  CUDA_OK(e, cudaMemcpyAsync(b.lut1.p, l1.data(), l1.size() * 8, cudaMemcpyHostToDevice, e->cs));
  CUDA_OK(e, cudaMemcpyAsync(b.lut2.p, l2.data(), l2.size() * 8, cudaMemcpyHostToDevice, e->cs));
  CUDA_OK(e, cudaStreamSynchronize(e->cs));
  b.cols1.assign(b.M1.c(), 0); b.cols2.assign(b.M2.c(), 0);
  for(unsigned i = 0; i < b.M1.c(); ++i) { b.cols1[i] = b.M1[i]; b.cols2[i] = b.M2[i]; }
  b.drawn = true;
  return JFGPU_OK;
}
// hash_pair<mer_dna>() (mer_dna_bloom_counter.hpp:22-27): two 64 x 2k matrices, randomize() only, the next draws of the stream
int bloom_draw(jfgpu_engine* e) {
  BloomState& b = e->bloom;
  if(b.drawn || b.mode == BLOOM_NONE) return JFGPU_OK;
  b.M1 = jfb::gf2_matrix(64, 2 * e->k); b.M1.randomize(e->rng);
  b.M2 = jfb::gf2_matrix(64, 2 * e->k); b.M2.randomize(e->rng);
  return bloom_upload_matrices(e);
}
BloomDev bloom_dev(const jfgpu_engine* e) {
  BloomDev d;
  memset(&d, 0, sizeof(d));
  const BloomState& b = e->bloom;
  // the PRIME pass of --if is not filtered (count_main.cc:288-295 builds that counter without a filter)
  if(b.mode == BLOOM_NONE || !b.drawn || (e->op == JFGPU_OP_PRIME && b.mode != BLOOM_COUNT)) return d;
  d.mode = b.mode; d.k = b.k; d.m = b.m; d.inv = b.inv;
  d.bits = b.bits.as<uint32_t>(); d.locks = b.locks.as<uint32_t>(); d.lock_mask = (uint32_t)(b.locks.bytes / 4 - 1);
  d.lut1 = b.lut1.as<uint64_t>(); d.lut2 = b.lut2.as<uint64_t>();
  return d;
}

int reset_carry(jfgpu_engine* e, cudaStream_t stream) {
  Carry c;
  c.state = e->format == 1 ? (0u | 4u) : (uint32_t)ST_L;    // FASTQ: header line expected, at a line start
  c.pad = 0;
  memset(c.sym, SYM_BREAK, sizeof(c.sym));
  // (stream ordered; source is copied synchronously into the driver's staging for pageable memory)
  CUDA_OK(e, cudaMemcpyAsync(e->carry[e->carry_cur].p, &c, sizeof(c), cudaMemcpyHostToDevice, stream));
  CUDA_OK(e, cudaStreamSynchronize(stream));
  return JFGPU_OK;
}

int read_stats(jfgpu_engine* e) {
  CUDA_OK(e, cudaMemcpyAsync(e->h_stats, e->stats.p, STAT_N * 8, cudaMemcpyDeviceToHost, e->cs));
  CUDA_OK(e, cudaStreamSynchronize(e->cs));
  return JFGPU_OK;
}

int insert_keys_into(jfgpu_engine* e, Table& t, const uint64_t* keys, const uint64_t* counts, uint64_t n, cudaStream_t stream) {
  if(n == 0) return JFGPU_OK;
  int rc = table_materialize(e, t, stream);
  if(rc) return rc;
  TableDev T = table_dev(e, t);
  const size_t smem = (size_t)e->nbytes * 256 * 8;
  const int grid = (int)std::min<uint64_t>((n + 255) / 256, (uint64_t)e->n_sm * 8);
  auto run = [&](auto kern) -> int {
    cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    kern<<<grid, 256, smem, stream>>>(T, t.lut.as<uint64_t>(), e->nbytes, keys, counts, n);
    return JFGPU_OK;
  };
  rc = e->kw == 4 ? run(wide_kernels().insert_keys)
                  : dispatch(e, e->kw, t.slot_bits, [&](auto KW, auto SB) -> int { return run(insert_keys_kernel<decltype(KW)::value, decltype(SB)::value>); });
  if(rc) return rc;
  JF_LAUNCHED();
  CUDA_OK(e, cudaGetLastError());
  return JFGPU_OK;
}

struct SegScratch {
  DevBuf keys, counts, sort_lo, n_out;
  uint64_t cap = 0;
};

int seg_alloc(jfgpu_engine* e, SegScratch& s, uint64_t cap) {
  s.cap = cap;
  CUDA_OK(e, s.keys.alloc(cap * 8 * e->kw));
  CUDA_OK(e, s.counts.alloc(cap * 8));
  CUDA_OK(e, s.n_out.alloc(8));
  CUDA_OK(e, s.sort_lo.alloc(cap * 8));
  return JFGPU_OK;
}

// Collect the records of local original positions [lo, hi) of table t; returns their number.
int collect_segment(jfgpu_engine* e, Table& t, SegScratch& s, uint64_t lo, uint64_t hi, uint64_t lower, uint64_t upper, uint64_t* n_rec) {
  CollectArgs a;
  memset(&a, 0, sizeof(a));
  a.T = table_dev(e, t);
  a.inv_lut = t.inv_lut.as<uint64_t>();
  a.nbytes = e->nbytes;
  a.seg_lo = lo; a.seg_hi = hi;
  a.scan_hi = std::min<uint64_t>(hi + t.margin, t.local_size + t.margin);
  a.lower = lower; a.upper = upper;
  a.hb = t.hb;
  a.out_keys = s.keys.as<uint64_t>(); a.out_counts = s.counts.as<uint64_t>();
  a.out_sort_lo = s.sort_lo.as<uint64_t>();
  a.out_sort_hi = nullptr;
  a.out_n = s.n_out.as<unsigned long long>();
  a.out_cap = s.cap;
  CUDA_OK(e, cudaMemsetAsync(s.n_out.p, 0, 8, e->cs));
  const size_t smem = (size_t)e->nbytes * 256 * 8;
  const uint64_t span = a.scan_hi - a.seg_lo;
  const int grid = (int)std::min<uint64_t>((span + 255) / 256, (uint64_t)e->n_sm * 16);
  auto run = [&](auto kern) -> int {
    cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    kern<<<grid, 256, smem, e->cs>>>(a);
    return JFGPU_OK;
  };
  int rc = e->kw == 4 ? run(wide_kernels().collect)
                      : dispatch(e, e->kw, t.slot_bits, [&](auto KW, auto SB) -> int { return run(collect_kernel<decltype(KW)::value, decltype(SB)::value>); });
  if(rc) return rc;
  JF_LAUNCHED();
  unsigned long long n = 0;
  CUDA_OK(e, cudaMemcpyAsync(&n, s.n_out.p, 8, cudaMemcpyDeviceToHost, e->cs));
  CUDA_OK(e, cudaStreamSynchronize(e->cs));
  if(n > s.cap) return fail(e, JFGPU_ERR_STATE, "internal: segment overflow in collect");
  *n_rec = n;
  return JFGPU_OK;
}

// local positions of a table collected (regrow) or dumped at once
uint64_t pick_segment(const Table& t) { return std::min<uint64_t>(t.local_size, (uint64_t)1 << 24); }

// While it lives, counts are added (JFGPU_OP_COUNT) whatever operation the counter is in: moving (key, count) pairs into a
// table, or loading a database, is plain addition.
struct ForceCount {
  jfgpu_engine* e; const uint32_t op;
  explicit ForceCount(jfgpu_engine* e_) : e(e_), op(e_->op) { e->op = JFGPU_OP_COUNT; }
  ~ForceCount() { e->op = op; }
};

// Turn to the other failure list (allocated on first use), so that the failures of a re-insertion are kept apart.
int flip_fail_list(jfgpu_engine* e) {
  const int next = e->fail_cur ^ 1;
  if(!e->fail_keys[next].p) CUDA_OK(e, make_all(need(e->fail_keys[next], e->fail_cap * 8 * e->kw), need(e->fail_counts[next], e->fail_cap * 8)));
  e->fail_cur = next;
  return JFGPU_OK;
}

// Move every (key, count) of the current table, plus `n_failed` entries of failure list
// `old_fail`, into a fresh table of 2^nl global slots hashed with M.
int rebuild_table(jfgpu_engine* e, unsigned nl, const jfb::gf2_matrix& M, int old_fail, uint64_t n_failed) {
  const ForceCount force_count(e);
  Table nt;
  int rc = table_setup(e, nt, nl, M, e->tab.max_reprobe);
  if(rc) return rc == JFGPU_ERR_NOMEM ? fail(e, JFGPU_ERR_FULL, "Hash full (" + e->err + ")") : rc;
  rc = table_zero(e, nt, false);
  if(rc) return rc;
  // distinct / reprobes statistics restart for the new table; STAT_INSERTED counts k-mer
  // occurrences and must not change
  unsigned long long inserted_before = 0, failed_before = 0;
  CUDA_OK(e, cudaMemcpyAsync(&inserted_before, e->stats.as<unsigned long long>() + STAT_INSERTED, 8, cudaMemcpyDeviceToHost, e->cs));
  CUDA_OK(e, cudaMemcpyAsync(&failed_before, e->stats.as<unsigned long long>() + STAT_FAILED, 8, cudaMemcpyDeviceToHost, e->cs));
  CUDA_OK(e, cudaStreamSynchronize(e->cs));
  CUDA_OK(e, cudaMemsetAsync(e->stats.as<unsigned long long>() + STAT_DISTINCT, 0, 8, e->cs));
  CUDA_OK(e, cudaMemsetAsync(e->stats.as<unsigned long long>() + STAT_REPROBES, 0, 8, e->cs));
  {
    SegScratch s;                // (goes at the end of this block, before the failed keys are inserted)
    const uint64_t seg = pick_segment(e->tab);
    rc = seg_alloc(e, s, seg + e->tab.margin + 8);
    for(uint64_t lo = 0; lo < e->tab.local_size && !rc; lo += seg) {
      uint64_t n = 0;
      rc = collect_segment(e, e->tab, s, lo, std::min(lo + seg, e->tab.local_size), 0, ~0ull, &n);
      if(!rc) rc = insert_keys_into(e, nt, s.keys.as<uint64_t>(), s.counts.as<uint64_t>(), n, e->cs);
    }
    cudaStreamSynchronize(e->cs);
  }
  if(rc) return rc;
  // the moved entries are not new k-mer occurrences; the failed ones (below) are.  A moved entry that found no slot in the
  // new table (a clipped reprobe limit) waits in the failure list like a key that never reached a table, and is counted
  // when the next table takes it: it leaves STAT_INSERTED now.
  unsigned long long failed_after = 0;
  CUDA_OK(e, cudaMemcpyAsync(&failed_after, e->stats.as<unsigned long long>() + STAT_FAILED, 8, cudaMemcpyDeviceToHost, e->cs));
  CUDA_OK(e, cudaStreamSynchronize(e->cs));
  failed_after = std::min<unsigned long long>(failed_after, e->fail_cap);
  if(failed_after > failed_before) {
    std::vector<uint64_t> waiting(failed_after - failed_before);
    CUDA_OK(e, cudaMemcpyAsync(waiting.data(), e->fail_counts[e->fail_cur].as<uint64_t>() + failed_before, waiting.size() * 8,
                               cudaMemcpyDeviceToHost, e->cs));
    CUDA_OK(e, cudaStreamSynchronize(e->cs));
    for(const uint64_t c : waiting) inserted_before -= c;
  }
  CUDA_OK(e, cudaMemcpyAsync(e->stats.as<unsigned long long>() + STAT_INSERTED, &inserted_before, 8, cudaMemcpyHostToDevice, e->cs));
  CUDA_OK(e, cudaStreamSynchronize(e->cs));
  if(n_failed) {
    rc = insert_keys_into(e, nt, e->fail_keys[old_fail].as<uint64_t>(), e->fail_counts[old_fail].as<uint64_t>(), n_failed, e->cs);
    cudaStreamSynchronize(e->cs);
    if(rc) return rc;
  }
  // (each table owns its counter-carry side table: the old one dies with the old slots)
  e->tab = std::move(nt);
  if(!e->part.pending) { part_configure(e); if(!e->part.P) e->part = PartState(); }
  return JFGPU_OK;
}

// hash_counter::handle_full_ary without doubling (hash_counter.hpp:187-192): the caller's hook writes the resident table out,
// the table is zeroed, the keys that found no slot go into the empty table, counting continues with the same geometry.
int spill_table(jfgpu_engine* e, uint64_t n_failed) {
  e->in_spill = true;
  const int hrc = e->spill_fn(e->spill_ctx, e);
  e->in_spill = false;
  if(hrc) return fail(e, JFGPU_ERR_SINK, "the spill hook failed (--disk: writing an intermediate file)");
  int rc = table_zero(e, e->tab, false);
  if(rc) return rc;
  unsigned long long* st = e->stats.as<unsigned long long>();
  CUDA_OK(e, cudaMemsetAsync(st + STAT_DISTINCT, 0, 8, e->cs));       // (statistics of the table restart; STAT_INSERTED counts occurrences and goes on)
  CUDA_OK(e, cudaMemsetAsync(st + STAT_REPROBES, 0, 8, e->cs));
  CUDA_OK(e, cudaMemsetAsync(st + STAT_OVERFLOWED, 0, 8, e->cs));
  CUDA_OK(e, cudaMemsetAsync(st + STAT_FAILED, 0, 8, e->cs));
  CUDA_OK(e, cudaStreamSynchronize(e->cs));
  const int old_fail = e->fail_cur;
  rc = flip_fail_list(e);                             // (failures of the re-insertion -- there should be none -- are kept apart)
  if(rc) return rc;
  {
    const ForceCount force_count(e);
    rc = insert_keys_into(e, e->tab, e->fail_keys[old_fail].as<uint64_t>(), e->fail_counts[old_fail].as<uint64_t>(), n_failed, e->cs);
  }
  if(rc) return rc;
  CUDA_OK(e, cudaStreamSynchronize(e->cs));       // (the keys that had found no slot are counted as inserted now, once)
  e->spills++;
  return JFGPU_OK;
}

// hash_counter::double_size (hash_counter.hpp:200-238): allocate a table twice as large with a
// freshly drawn matrix, re-insert every (key, count) of the old one, then the keys that failed.
int regrow(jfgpu_engine* e) {
  for(;;) {
    int rc = read_stats(e);
    if(rc) return rc;
    if(e->h_stats[STAT_OVF_FULL]) return fail(e, JFGPU_ERR_FULL, "counter overflow side table is full");
    const uint64_t n_failed = e->h_stats[STAT_FAILED];
    if(n_failed == 0) return JFGPU_OK;
    if(e->h_stats[STAT_FAIL_DROPPED]) return fail(e, JFGPU_ERR_FULL, "Hash full (too many keys failed before the table could be doubled)");
    const unsigned kbits = 2 * e->k;
    if(!e->p.allow_regrow || e->shard_bits || (kbits < 64 && e->tab.size >= ((uint64_t)1 << kbits))) {
      if(e->spill_fn) { rc = spill_table(e, n_failed); if(rc) return rc; continue; }
      return fail(e, JFGPU_ERR_FULL, "Hash full");
    }
    const unsigned nl = e->tab.lsize + 1;
    jfb::gf2_matrix M = draw_matrix(e, (uint64_t)1 << nl, nl);
    const int old_fail = e->fail_cur;
    rc = flip_fail_list(e);
    if(rc) return rc;
    CUDA_OK(e, cudaMemsetAsync(e->stats.as<unsigned long long>() + STAT_FAILED, 0, 8, e->cs));
    rc = rebuild_table(e, nl, M, old_fail, n_failed);
    if(rc == JFGPU_ERR_FULL && e->spill_fn) {          // no memory for the doubled table: dump and zero this one instead
      e->fail_cur = old_fail;
      CUDA_OK(e, cudaMemcpyAsync(e->stats.as<unsigned long long>() + STAT_FAILED, &n_failed, 8, cudaMemcpyHostToDevice, e->cs));
      CUDA_OK(e, cudaStreamSynchronize(e->cs));
      rc = spill_table(e, n_failed);
      if(rc) return rc;
      continue;
    }
    if(rc) return rc;
    e->regrows++;
  }
}

// Direct-indexing regime (table as large as the key space, no reprobing).  The reference
// cannot chain "large" continuation entries there, so a counter that outgrows val_len bits
// makes hash_counter::double_size build a new array with val_len + 1 -- and, the size being
// 4^k, with the IDENTITY matrix (hash_counter.hpp:205-212, large_hash_array.hpp:992-1002).
// The observable result is: val_len = bits of the largest count, identity hash.
int direct_index_fixup(jfgpu_engine* e) {
  const unsigned kbits = 2 * e->k;
  if(e->tab.lsize < kbits || e->shard_bits) return JFGPU_OK;
  CUDA_OK(e, cudaMemsetAsync(e->stats.as<unsigned long long>() + STAT_MAXCOUNT, 0, 8, e->cs));
  TableDev T = table_dev(e, e->tab);
  const uint64_t ns = e->tab.local_size + e->tab.margin;
  const int grid = (int)std::min<uint64_t>((ns + 255) / 256, (uint64_t)e->n_sm * 16);
  switch(e->tab.slot_bits) {
  case 32:  max_count_kernel<32><<<grid, 256, 0, e->cs>>>(T, ns); break;
  case 64:  max_count_kernel<64><<<grid, 256, 0, e->cs>>>(T, ns); break;
  default:  max_count_kernel<128><<<grid, 256, 0, e->cs>>>(T, ns); break;
  }
  JF_LAUNCHED();
  int rc = read_stats(e);
  if(rc) return rc;
  const uint64_t maxc = e->h_stats[STAT_MAXCOUNT];
  if(e->eff_val_len < 64 && (maxc >> e->eff_val_len) != 0) {
    e->eff_val_len = bitsize(maxc);
    if(!e->tab.M.is_identity()) {
      rc = rebuild_table(e, e->tab.lsize, jfb::gf2_matrix::identity(kbits), 0, 0);
      if(rc) return rc;
    }
  }
  return JFGPU_OK;
}

// fold the per-launch event pairs into kernel_ms (the stream must be idle)
void resolve_kernel_events(jfgpu_engine* e) {
  for(size_t i = 0; i + 1 < e->kev_used; i += 2) {
    float ms = 0;
    if(cudaEventElapsedTime(&ms, e->kev[i], e->kev[i + 1]) == cudaSuccess) { e->kernel_ms += ms; e->kernel_launches++; }
    else cudaGetLastError();
  }
  e->kev_used = 0;
}

int check_after_batches(jfgpu_engine* e) {
  int rc = read_stats(e);
  if(rc) return rc;
  if(e->h_stats[STAT_OVF_FULL]) return fail(e, JFGPU_ERR_FULL, "counter overflow side table is full");
  if(e->h_stats[STAT_FAILED]) {
    // records staged against the CURRENT geometry must reach the table before it is rebuilt: the drain copes
    // with a doubling in its middle (old inverse tables + rehash kernel), a plain regrow() would not
    if(e->part.pending) {
      rc = part_drain(e, e->cs);
      if(rc) return rc;
      rc = read_stats(e);
      if(rc) return rc;
      if(!e->h_stats[STAT_FAILED]) return JFGPU_OK;
    }
    return regrow(e);
  }
  return JFGPU_OK;
}

// A spill hook is set on an engine that inserts on a caller's stream (jfgpu_insert_keys, jfgpu_shard_unpack): once the work
// enqueued on `st` is done, keys that found no slot spill the table now, behind the drain of the pending region records, so
// that the failure list holds at most what the next slice adds (one failure group) when the slice begins.
int spill_if_failed(jfgpu_engine* e, cudaStream_t st) {
  CUDA_OK(e, cudaStreamSynchronize(st));
  CUDA_OK(e, cudaMemcpyAsync(e->h_stats + STAT_FAILED, e->stats.as<unsigned long long>() + STAT_FAILED, 8, cudaMemcpyDeviceToHost, e->cs));
  CUDA_OK(e, cudaStreamSynchronize(e->cs));
  return e->h_stats[STAT_FAILED] ? check_after_batches(e) : JFGPU_OK;
}

}  // namespace

// =======================================================================================
// C ABI
// =======================================================================================
extern "C" {

const char* jfgpu_version(void) { return "jellyfish-b200 0.1 (sm_90a)"; }
uint64_t jfgpu_kernel_launches(void) { return g_launches.load(); }
#if JF_K1_PROF
// the instrumented build only (scripts/k1_phases.py): copy out the phase counters of the FAST K1 kernels of the current
// device, then zero them
int jfgpu_k1_prof(unsigned long long* out, int n) {
  if(n != jfk::K1P_WORDS) return JFGPU_ERR_ARG;
  static const unsigned long long zero[jfk::K1P_WORDS] = {};
  if(cudaDeviceSynchronize() != cudaSuccess || cudaMemcpyFromSymbol(out, jfk::k1_prof_acc, sizeof(zero)) != cudaSuccess ||
     cudaMemcpyToSymbol(jfk::k1_prof_acc, zero, sizeof(zero)) != cudaSuccess) return JFGPU_ERR_CUDA;
  return JFGPU_OK;
}
#endif
const char* jfgpu_last_error(jfgpu_handle h) { return h ? h->err.c_str() : g_create_error.c_str(); }

void* jfgpu_host_alloc(size_t bytes) { void* p = nullptr; if(cudaHostAlloc(&p, bytes, cudaHostAllocDefault) != cudaSuccess) { cudaGetLastError(); return nullptr; } return p; }
void jfgpu_host_free(void* p) { if(p) cudaFreeHost(p); }
int jfgpu_memcpy_h2d(void* dev_dst, const void* host_src, size_t bytes, void* stream) {
  if(cudaMemcpyAsync(dev_dst, host_src, bytes, cudaMemcpyHostToDevice, (cudaStream_t)stream) != cudaSuccess) { cudaGetLastError(); return JFGPU_ERR_CUDA; }
  return JFGPU_OK;
}

int jfgpu_reference_matrix(uint32_t r, uint32_t c, uint32_t skip, uint64_t* cols) {
  if(r == 0 || r > 64 || c == 0 || c > 256 || !cols) return JFGPU_ERR_ARG;
  jfb::glibc_random rng;
  jfb::gf2_matrix res;
  for(uint32_t i = 0; i <= skip; ++i) { jfb::gf2_matrix m(r, c); res = m.randomize_pseudo_inverse(rng); }
  for(uint32_t i = 0; i < c; ++i) cols[i] = res[i];
  return JFGPU_OK;
}

int jfgpu_create(const jfgpu_params* params, jfgpu_handle* out) {
  if(!params || !out) return fail(nullptr, JFGPU_ERR_ARG, "null argument");
  if(params->struct_size != sizeof(jfgpu_params)) return fail(nullptr, JFGPU_ERR_ARG, "jfgpu_params size mismatch");
  if(params->k < 1 || params->k > 128) return fail(nullptr, JFGPU_ERR_ARG, "mer length must be in [1, 128]");
  if(params->size == 0) return fail(nullptr, JFGPU_ERR_ARG, "size must be positive");
  uint32_t ns = params->n_shards ? params->n_shards : 1;
  if(ns & (ns - 1)) return fail(nullptr, JFGPU_ERR_ARG, "n_shards must be a power of two");
  if(params->shard_index >= ns) return fail(nullptr, JFGPU_ERR_ARG, "shard_index out of range");
  if(params->max_reprobe > 255) return fail(nullptr, JFGPU_ERR_ARG, "max_reprobe must be <= 255");
  if(params->k > 64 && (params->bloom_counter || params->bf_size))
    return fail(nullptr, JFGPU_ERR_ARG, "Bloom filters and counters take mer lengths up to 64");
  if(params->k > 64 && ns > 8) return fail(nullptr, JFGPU_ERR_ARG, "sharded counting of mer lengths over 64 takes at most 8 shards");

  int ndev = 0;
  if(cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
    cudaGetLastError();
    return fail(nullptr, JFGPU_ERR_CUDA, "no CUDA device: the jellyfish-b200 engine has no CPU fallback");
  }
  if(params->device < 0 || params->device >= ndev) return fail(nullptr, JFGPU_ERR_ARG, "invalid device ordinal");

  jfgpu_engine* e = new jfgpu_engine;
  e->p = *params;
  e->p.n_shards = ns;
  e->device = params->device;
  e->k = params->k;
  e->kw = params->k > 64 ? 4 : params->k > 32 ? 2 : 1;
  e->nbytes = (2 * params->k + 7) / 8;
  e->eff_val_len = params->counter_len;
  e->shard_bits = ceil_log2(ns);
  auto bail = [&](int code) { g_create_error = e->err; jfgpu_destroy(e); return code; };

  cudaError_t c;
  if((c = cudaSetDevice(e->device)) != cudaSuccess) { e->err = cudaGetErrorString(c); return bail(JFGPU_ERR_CUDA); }
  cudaDeviceProp prop;
  if((c = cudaGetDeviceProperties(&prop, e->device)) != cudaSuccess) { e->err = cudaGetErrorString(c); return bail(JFGPU_ERR_CUDA); }
  if(prop.major != 9 || prop.minor != 0) { e->err = "this engine is built for sm_90a (Hopper) only"; return bail(JFGPU_ERR_CUDA); }
  e->n_sm = prop.multiProcessorCount;
  if(e->cs.create() != cudaSuccess || e->hs.create() != cudaSuccess) { e->err = "stream creation failed"; return bail(JFGPU_ERR_CUDA); }
  const unsigned untimed = cudaEventDisableTiming;
  if(make_all(need(e->ev_t0, cudaEventDefault), need(e->ev_t1, cudaEventDefault), need(e->ev_watch[0], untimed), need(e->ev_watch[1], untimed),
              need(e->ev_copied[0], untimed), need(e->ev_copied[1], untimed), need(e->ev_done[0], untimed), need(e->ev_done[1], untimed)) != cudaSuccess) {
    e->err = "event creation failed";
    return bail(JFGPU_ERR_CUDA);
  }

  if(params->bloom_counter) {
    // `jellyfish bc`: no hash table at all; the two hash matrices are the FIRST draws of the random stream (bc_main.cc:103-106)
    if(make_all(need(e->stats, STAT_N * 8), need(e->carry[0], sizeof(Carry)), need(e->carry[1], sizeof(Carry)), need(e->h_stats, STAT_N * 8),
                need(e->h_watch, 16)) != cudaSuccess) { e->err = "device allocation failed"; return bail(JFGPU_ERR_NOMEM); }
    cudaMemsetAsync(e->stats.p, 0, STAT_N * 8, e->cs);
    memset(e->h_stats, 0, STAT_N * 8);
    e->batch_bytes = params->max_batch_bytes ? (size_t)((params->max_batch_bytes + 15) & ~(uint64_t)15) : ((size_t)64 << 20);
    e->tab.slot_bits = 64; e->tab.lsize = 0; e->tab.size = 0;
    int rc0 = bloom_setup(e, BLOOM_COUNT, params->bf_size, params->bf_fp);
    if(!rc0) rc0 = bloom_draw(e);
    if(!rc0) rc0 = reset_carry(e, e->cs);
    if(rc0) return bail(rc0);
    *out = e;
    return JFGPU_OK;
  }

  // table geometry: size rounded up to a power of two, clipped to 4^k (large_hash_array.hpp:992-1002,150-153)
  const unsigned kbits = 2 * e->k;
  uint64_t req = params->size;
  if(kbits < 64 && req > ((uint64_t)1 << kbits)) req = (uint64_t)1 << kbits;
  const unsigned lsize = ceil_log2(req);
  if(lsize < e->shard_bits) { e->err = "table smaller than the number of shards"; return bail(JFGPU_ERR_ARG); }
  for(uint32_t i = 0; i < params->matrix_skip; ++i) (void)draw_matrix(e, params->size, lsize);
  jfb::gf2_matrix M = draw_matrix(e, params->size, lsize);

  // side structures
  e->batch_bytes = params->max_batch_bytes ? (size_t)((params->max_batch_bytes + 15) & ~(uint64_t)15) : ((size_t)64 << 20);
  // The failure counter is read one group late: the list holds the failed keys of two groups, and of one deferred list of
  // a write-only drain (part_drain: a group's deferred records run after the next group; at most WIN_DEF_CAP records and
  // at most a group).
  e->fail_group = e->batch_bytes;
  e->fail_cap = 2 * e->fail_group + std::min<uint64_t>(WIN_DEF_CAP, e->fail_group);
  if(make_all(need(e->stats, STAT_N * 8), need(e->carry[0], sizeof(Carry)), need(e->carry[1], sizeof(Carry)),
              need(e->fail_keys[0], e->fail_cap * 8 * e->kw), need(e->fail_counts[0], e->fail_cap * 8), need(e->h_stats, STAT_N * 8),
              need(e->h_watch, 16)) != cudaSuccess) { e->err = "device allocation failed"; return bail(JFGPU_ERR_NOMEM); }
  cudaMemsetAsync(e->stats.p, 0, STAT_N * 8, e->cs);
  memset(e->h_stats, 0, STAT_N * 8);
  int rc = table_setup(e, e->tab, lsize, M, params->max_reprobe);
  if(rc) return bail(rc);
  part_configure(e);
  // count --bf-size: mer_dna_bloom_filter(bf_fp, bf_size) in front of the table (count_main.cc:317-321); its matrices are
  // drawn when the first unprimed text arrives.  A shard's filter holds the keys it owns, about 1/n_shards of them: it is
  // sized for that share of the expected number, so its false positive rate is that of the single filter.
  if(params->bf_size) { rc = bloom_setup(e, BLOOM_FILTER, (params->bf_size + ns - 1) / ns, params->bf_fp); if(rc) return bail(rc); }
  rc = table_zero(e, e->tab, lazy_zero_ok(e));
  if(rc) return bail(rc);
  rc = reset_carry(e, e->cs);
  if(rc) return bail(rc);
  *out = e;
  return JFGPU_OK;
}

void jfgpu_destroy(jfgpu_handle e) {
  if(!e) return;
  cudaSetDevice(e->device);
  if(e->cs) cudaStreamSynchronize(e->cs);
  if(e->hs) cudaStreamSynchronize(e->hs);
  delete e;                      // (every buffer, event and stream is released by its owner, the streams last)
}

static void sam_begin(jfgpu_engine::SamState& s, uint32_t form) {
  s.form = form; s.tail.clear(); s.tail_dev_len = 0;
  s.bam_phase = 0; s.bam_refs = 0; s.bam_skip = 0; s.done_off = 0;
}

static int begin_feed(jfgpu_engine* e, uint32_t flags, int first_byte, cudaStream_t st) {
  if((flags & TEXT_FLAGS) == TEXT_FLAGS || ((flags & TEXT_FLAGS) && (flags & SAM_FLAGS)))
    return fail(e, JFGPU_ERR_ARG, "JFGPU_FORMAT_FASTA, _FASTQ, _SAM and _BAM exclude each other");
  if(flags & JFGPU_FILE_BEGIN) {
    // mer_overlap_sequence_parser.hpp:134-148: the first byte selects the format, unless the caller gives it (a share that
    // starts in the middle of a file, or SAM / BAM)
    const uint32_t form = flags & JFGPU_FORMAT_BAM ? 2 : flags & JFGPU_FORMAT_SAM ? 1 : 0;
    if(!form && !(flags & TEXT_FLAGS) && first_byte >= 0 && first_byte != '>' && first_byte != '@') return fail(e, JFGPU_ERR_FORMAT, "Unsupported format");
    // SAM and BAM records reach the extraction kernels as 4-line FASTQ
    e->format = form || (flags & JFGPU_FORMAT_FASTQ) || (!(flags & JFGPU_FORMAT_FASTA) && first_byte == '@') ? 1 : 0;
    sam_begin(e->sam, form);
    int rc = reset_carry(e, st);
    if(rc) return rc;
    e->in_file = true;
  }
  return JFGPU_OK;
}

// begin_feed of text in device memory: its first byte is read back to select the format
static int begin_device_feed(jfgpu_engine* e, uint32_t flags, const void* dev_bytes, size_t n, cudaStream_t st) {
  int first = -1;
  if((flags & JFGPU_FILE_BEGIN) && n) {
    unsigned char b = 0;
    CUDA_OK(e, cudaMemcpyAsync(&b, dev_bytes, 1, cudaMemcpyDeviceToHost, st));
    CUDA_OK(e, cudaStreamSynchronize(st));
    first = b;
  }
  return begin_feed(e, flags, first, st);
}

// One batch of host text through the next staging buffer: copied on the copy stream, run on the compute stream once the
// copy is done.  The caller has waited for ev_done of that buffer (the previous batch that used it has finished).
// The batch is bytes [off, off + len) of the n bytes of this feed.  A batch that still ends on '\r' (next_batch_len could not
// cut in front of the run: the run fills the batch, or follows its first byte) gets the byte that ends the run staged behind
// it as one byte of look-ahead, so that the device drops the run when a '\n' ends it and resets the window when a base does,
// as it would with the whole text in view.  A run that reaches the end of the data is a line end.
static int run_staged(jfgpu_engine* e, const char* bytes, size_t off, size_t len, size_t n, K1Use use) {
  const int s = e->stage_cur;
  CUDA_OK(e, cudaMemcpyAsync(e->stage[s].p, bytes + off, len, cudaMemcpyHostToDevice, e->hs));
  size_t n_look = len;
  if(len && off + len < n && bytes[off + len - 1] == '\r') {
    size_t q = off + len;
    while(q < n && bytes[q] == '\r') ++q;
    if(q < n) {
      e->stage_look[s] = (uint8_t)bytes[q];
      CUDA_OK(e, cudaMemcpyAsync(e->stage[s].as<uint8_t>() + len, &e->stage_look[s], 1, cudaMemcpyHostToDevice, e->hs));
      n_look = len + 1;
    }
  }
  CUDA_OK(e, cudaEventRecord(e->ev_copied[s], e->hs));
  CUDA_OK(e, cudaStreamWaitEvent(e->cs, e->ev_copied[s], 0));
  const int rc = run_batch(e, e->stage[s].as<uint8_t>(), len, n_look, e->cs, use);
  if(rc) return rc;
  CUDA_OK(e, cudaEventRecord(e->ev_done[s], e->cs));
  e->stage_cur ^= 1;
  return JFGPU_OK;
}

static int end_feed(jfgpu_engine* e, uint32_t flags, cudaStream_t st) {
  if(flags & JFGPU_FILE_END) {
    // no k-mer spans two files: mer_overlap_sequence_parser.hpp:111
    e->format = 0; e->sam.form = 0;
    int rc = reset_carry(e, st);
    if(rc) return rc;
    e->in_file = false;
  }
  return JFGPU_OK;
}

// ---- SAM and BAM input (JFGPU_FORMAT_SAM / _BAM): batches of whole records are rewritten as FASTQ by the kernels of
// jf_sam.cu and counted as FASTQ.  The FASTQ of a batch is whole records, so the -Q rule "a K1 batch ends on a record
// boundary" holds by construction.
enum : uint32_t { BAM_MAGIC = 0, BAM_NREF = 1, BAM_REF = 2, BAM_RECORDS = 3 };

static int sam_alloc(jfgpu_engine* e) {
  jfgpu_engine::SamState& s = e->sam;
  if(!e->stage[0].p) CUDA_OK(e, e->stage[0].alloc(e->batch_bytes + 64));
  if(s.out.p) return JFGPU_OK;
  s.in_cap = std::max<size_t>(std::min<size_t>(e->batch_bytes / 2, (size_t)1 << 30) & ~(size_t)15, 64);
  const size_t max_recs = jfsam::max_bam_records(s.in_cap);
  if(make_all(need(s.out, 2 * s.in_cap + 64), need(s.scratch, jfsam::scratch_bytes(s.in_cap)), need(s.res, sizeof(jfsam::Result)),
              need(s.offs, max_recs * 4), need(s.tail_dev, s.in_cap + 64), need(s.h_res, sizeof(jfsam::Result)),
              need(s.h_offs, max_recs * 4)) != cudaSuccess)
    return fail(e, JFGPU_ERR_NOMEM, "Failed to allocate the SAM/BAM batch buffers");
  return JFGPU_OK;
}

// input bytes of the next batch: its FASTQ must fit one K1 batch and the record pool
static size_t sam_batch_cap(const jfgpu_engine* e) {
  return std::max<size_t>(std::min(e->sam.in_cap, part_cap_len(e, 2 * e->sam.in_cap) / 2) & ~(size_t)15, 16);
}

// Transcode the batch [dev, dev + n) that starts at byte `at` of the file (BAM: its n_recs records at the offsets in
// sam.offs) on `st` and count the FASTQ it becomes.  *used = the input bytes transcoded (SAM: through the last newline, all
// of them when `final`).
static int sam_run(jfgpu_engine* e, cudaStream_t st, const uint8_t* dev, size_t n, bool final, uint32_t n_recs, uint64_t at, size_t* used) {
  jfgpu_engine::SamState& s = e->sam;
  const int launches = s.form == 2
      ? jfsam::bam_transcode(dev, n, s.offs.as<uint32_t>(), n_recs, s.out.as<uint8_t>(), s.scratch.p, s.in_cap, s.res.as<jfsam::Result>(), st)
      : jfsam::sam_transcode(dev, n, final, s.out.as<uint8_t>(), s.scratch.p, s.in_cap, s.res.as<jfsam::Result>(), st);
  g_launches.fetch_add(launches, std::memory_order_relaxed);
  CUDA_OK(e, cudaGetLastError());
  CUDA_OK(e, cudaMemcpyAsync(s.h_res, s.res.p, sizeof(jfsam::Result), cudaMemcpyDeviceToHost, st));
  CUDA_OK(e, cudaStreamSynchronize(st));
  const jfsam::Result r = *s.h_res;
  if(r.err) {
    const unsigned long long v = ~r.err;
    static const char* const what[] = { "", "fewer than 11 fields", "SEQ and QUAL of different lengths", "its fields run past its block_size" };
    return fail(e, JFGPU_ERR_FORMAT, std::string(s.form == 2 ? "Invalid BAM record at byte " : "Invalid SAM line at byte ") +
                std::to_string(at + (v >> 2)) + " of the " + (s.form == 2 ? "inflated " : "") + "file: " + what[v & 3]);
  }
  *used = s.form == 2 ? n : (size_t)r.consumed;
  if(!r.out_bytes) return JFGPU_OK;
  if(e->stage_out) {                          // jfgpu_sam_stage: the FASTQ goes to the caller, nothing is counted
    if(r.out_bytes > e->stage_out_cap - e->stage_out_len)
      return fail(e, JFGPU_ERR_ARG, "jfgpu_sam_stage: the FASTQ of the input does not fit out_cap (" + std::to_string(e->stage_out_cap) + " bytes)");
    CUDA_OK(e, cudaMemcpyAsync(e->stage_out + e->stage_out_len, s.out.p, r.out_bytes, cudaMemcpyDeviceToDevice, st));
    e->stage_out_len += r.out_bytes;
    return JFGPU_OK;
  }
  if((e->p.allow_regrow || e->spill_fn) && e->tab.slots.p) {            // as jfgpu_feed: a failed insertion regrows first
    CUDA_OK(e, cudaMemcpyAsync(e->h_stats + STAT_FAILED, e->stats.as<unsigned long long>() + STAT_FAILED, 8, cudaMemcpyDeviceToHost, e->cs));
    CUDA_OK(e, cudaStreamSynchronize(e->cs));
    if(e->h_stats[STAT_FAILED]) { const int rc = check_after_batches(e); if(rc) return rc; }
  }
  return run_batch(e, s.out.as<uint8_t>(), r.out_bytes, r.out_bytes, st, K1_COUNT);
}

// a batch of host bytes through staging buffer 0 (free again: the previous batch was transcoded and read back)
static int sam_stage(jfgpu_engine* e, const char* src, size_t len, bool final, uint32_t n_recs) {
  jfgpu_engine::SamState& s = e->sam;
  CUDA_OK(e, cudaMemcpyAsync(e->stage[0].p, src, len, cudaMemcpyHostToDevice, e->hs));
  if(n_recs) CUDA_OK(e, cudaMemcpyAsync(s.offs.p, s.h_offs, (size_t)n_recs * 4, cudaMemcpyHostToDevice, e->hs));
  CUDA_OK(e, cudaEventRecord(e->ev_copied[0], e->hs));
  CUDA_OK(e, cudaStreamWaitEvent(e->cs, e->ev_copied[0], 0));
  size_t used = 0;
  const int rc = sam_run(e, e->cs, e->stage[0].as<uint8_t>(), len, final, n_recs, s.done_off, &used);
  if(rc) return rc;
  s.done_off += len;
  return JFGPU_OK;
}

static int sam_too_long(jfgpu_engine* e) {
  return fail(e, JFGPU_ERR_FORMAT, "a SAM line or BAM record is longer than the staging buffer (max_batch_bytes / 2)");
}

// SAM text in host memory: whole lines per batch, the incomplete last line kept for the next feed
static int sam_feed_host(jfgpu_engine* e, const char* bytes, size_t n, bool end) {
  jfgpu_engine::SamState& s = e->sam;
  const size_t cap = sam_batch_cap(e);
  size_t pos = 0;
  int rc;
  if(!s.tail.empty()) {                       // the line the previous feed cut, completed
    const char* nl = n ? (const char*)memchr(bytes, '\n', n) : nullptr;
    pos = nl ? (size_t)(nl - bytes) + 1 : n;
    if(s.tail.size() + pos > cap) return sam_too_long(e);
    s.tail.append(bytes, pos);
    if(!nl && !end) return JFGPU_OK;
    if((rc = sam_stage(e, s.tail.data(), s.tail.size(), end && pos == n, 0))) return rc;
    s.tail.clear();
  }
  size_t stop = n;
  if(!end) {
    const char* nl = pos < n ? (const char*)memrchr(bytes + pos, '\n', n - pos) : nullptr;
    stop = nl ? (size_t)(nl - bytes) + 1 : pos;
  }
  while(pos < stop) {
    size_t len = std::min(cap, stop - pos);
    if(pos + len < stop) {
      const char* nl = (const char*)memrchr(bytes + pos, '\n', len);
      if(!nl) return sam_too_long(e);
      len = (size_t)(nl - (bytes + pos)) + 1;
    }
    if((rc = sam_stage(e, bytes + pos, len, end && pos + len == n, 0))) return rc;
    pos += len;
  }
  if(n - pos > cap) return sam_too_long(e);
  s.tail.assign(bytes + pos, n - pos);
  return JFGPU_OK;
}

static uint32_t le32(const char* p) { uint32_t v; memcpy(&v, p, 4); return v; }

// BAM header (SAM specification 4.2): magic and l_text, then the text; n_ref; for every reference l_name, then the name and
// l_ref.  The text and the names are passed over.
static int bam_header_field(jfgpu_engine* e, const char* p) {
  jfgpu_engine::SamState& s = e->sam;
  if(s.bam_phase == BAM_MAGIC) {
    if(memcmp(p, "BAM\1", 4) != 0) return fail(e, JFGPU_ERR_FORMAT, "Invalid BAM magic");
    s.bam_skip = le32(p + 4); s.bam_phase = BAM_NREF;
  } else if(s.bam_phase == BAM_NREF) {
    const int32_t nr = (int32_t)le32(p);
    if(nr < 0) return fail(e, JFGPU_ERR_FORMAT, "Invalid BAM header: negative number of references");
    s.bam_refs = (uint32_t)nr; s.bam_phase = nr ? BAM_REF : BAM_RECORDS;
  } else {
    s.bam_skip = (uint64_t)le32(p) + 4;
    if(--s.bam_refs == 0) s.bam_phase = BAM_RECORDS;
  }
  return JFGPU_OK;
}

// bytes of the record at byte `at` of the file, whose block_size field is at p
static int bam_record_len(jfgpu_engine* e, const char* p, size_t cap, uint64_t at, size_t* len) {
  *len = 4 + (size_t)le32(p);
  if(*len < 36)
    return fail(e, JFGPU_ERR_FORMAT, "Invalid BAM record at byte " + std::to_string(at) + " of the inflated file: block_size " +
                std::to_string(*len - 4) + " is below the 32 bytes of its fixed fields");
  return *len > cap ? sam_too_long(e) : JFGPU_OK;
}

// The inflated BAM stream in host memory: the host walks the header and the block_size chain; the records go to the device in
// batches with their offsets.  A header field or record the feed cuts is kept for the next feed.
static int bam_feed_host(jfgpu_engine* e, const char* bytes, size_t n, bool end) {
  jfgpu_engine::SamState& s = e->sam;
  const size_t cap = sam_batch_cap(e);
  size_t pos = 0;
  int rc;
  while(true) {
    if(s.bam_skip) {
      const size_t t = (size_t)std::min<uint64_t>(s.bam_skip, n - pos);
      s.bam_skip -= t; pos += t; s.done_off += t;
      if(s.bam_skip) break;
      continue;
    }
    const size_t head = s.bam_phase == BAM_MAGIC ? 8 : 4;     // the bytes that give a piece's length
    if(!s.tail.empty()) {                     // a piece the previous feed cut
      size_t t = std::min(n - pos, head > s.tail.size() ? head - s.tail.size() : 0);
      s.tail.append(bytes + pos, t); pos += t;
      if(s.tail.size() < head) break;
      size_t len = head;
      if(s.bam_phase == BAM_RECORDS && (rc = bam_record_len(e, s.tail.data(), cap, s.done_off, &len))) return rc;
      t = std::min(n - pos, len - s.tail.size());
      s.tail.append(bytes + pos, t); pos += t;
      if(s.tail.size() < len) break;
      if(s.bam_phase == BAM_RECORDS) { s.h_offs[0] = 0; rc = sam_stage(e, s.tail.data(), len, false, 1); }
      else { rc = bam_header_field(e, s.tail.data()); s.done_off += len; }
      if(rc) return rc;
      s.tail.clear();
      continue;
    }
    if(pos == n) break;
    if(s.bam_phase != BAM_RECORDS) {
      if(n - pos < head) { s.tail.assign(bytes + pos, n - pos); pos = n; break; }
      if((rc = bam_header_field(e, bytes + pos))) return rc;
      pos += head; s.done_off += head;
      continue;
    }
    // whole records in place, at most `cap` bytes per batch
    size_t run = pos;
    uint32_t nr = 0;
    while(n - pos >= 4) {
      size_t len = 4 + (size_t)le32(bytes + pos);
      if(len < 36 || len > cap) {           // the records in front of it come first: a bad one among them is the first error
        if(nr && (rc = sam_stage(e, bytes + run, pos - run, false, nr))) return rc;
        return bam_record_len(e, bytes + pos, cap, s.done_off, &len);
      }
      if(n - pos < len) break;
      if(pos + len - run > cap) {
        if((rc = sam_stage(e, bytes + run, pos - run, false, nr))) return rc;
        run = pos; nr = 0;
      }
      s.h_offs[nr++] = (uint32_t)(pos - run);
      pos += len;
    }
    if(nr && (rc = sam_stage(e, bytes + run, pos - run, false, nr))) return rc;
    s.tail.assign(bytes + pos, n - pos);
    break;
  }
  if(end && (s.bam_phase != BAM_RECORDS || s.bam_skip || !s.tail.empty()))
    return fail(e, JFGPU_ERR_FORMAT, s.bam_phase != BAM_RECORDS || s.bam_skip ? std::string("Truncated BAM header")
                                     : "Truncated BAM record at byte " + std::to_string(s.done_off) + " of the inflated file");
  return JFGPU_OK;
}

// SAM text in device memory: the kernels find the last newline of every batch; the incomplete last line of the feed is kept
// in sam.tail_dev and completed from the front of the next one
static int sam_feed_device(jfgpu_engine* e, const uint8_t* dev, size_t n, bool end, cudaStream_t st) {
  jfgpu_engine::SamState& s = e->sam;
  const size_t cap = sam_batch_cap(e);
  size_t pos = 0, used = 0;
  int rc;
  if(s.tail_dev_len) {
    const size_t take = s.tail_dev_len < cap ? std::min(n, cap - s.tail_dev_len) : 0;
    if(take < n && !take) return sam_too_long(e);
    CUDA_OK(e, cudaMemcpyAsync(s.tail_dev.as<uint8_t>() + s.tail_dev_len, dev, take, cudaMemcpyDeviceToDevice, st));
    const bool fin = end && take == n;
    if((rc = sam_run(e, st, s.tail_dev.as<uint8_t>(), s.tail_dev_len + take, fin, 0, s.done_off, &used))) return rc;
    if(!used) {                               // no newline yet
      if(take < n) return sam_too_long(e);
      s.tail_dev_len += take;
      return JFGPU_OK;
    }
    pos = used - s.tail_dev_len; s.done_off += used; s.tail_dev_len = 0;
  }
  while(pos < n) {
    const size_t len = std::min(cap, n - pos);
    if((rc = sam_run(e, st, dev + pos, len, end && pos + len == n, 0, s.done_off, &used))) return rc;
    if(!used) {
      if(pos + len < n) return sam_too_long(e);
      break;
    }
    pos += used; s.done_off += used;
  }
  if(pos < n) {
    CUDA_OK(e, cudaMemcpyAsync(s.tail_dev.p, dev + pos, n - pos, cudaMemcpyDeviceToDevice, st));
    s.tail_dev_len = n - pos;
  }
  return JFGPU_OK;
}

// jfgpu_feed / jfgpu_feed_device of a SAM or BAM file
static int sam_feed(jfgpu_engine* e, const void* data, size_t n, uint32_t flags, bool device, cudaStream_t st) {
  const uint32_t form = flags & JFGPU_FORMAT_BAM ? 2 : flags & JFGPU_FORMAT_SAM ? 1 : 0;
  if(flags & TEXT_FLAGS) return fail(e, JFGPU_ERR_ARG, "JFGPU_FORMAT_FASTA, _FASTQ, _SAM and _BAM exclude each other");
  if((flags & SAM_FLAGS) == SAM_FLAGS) return fail(e, JFGPU_ERR_ARG, "JFGPU_FORMAT_SAM and JFGPU_FORMAT_BAM exclude each other");
  if(!(flags & JFGPU_FILE_BEGIN) && form && form != e->sam.form) return fail(e, JFGPU_ERR_ARG, "the format flag differs from the one the file began with");
  if(device && (flags & JFGPU_FILE_BEGIN ? form : e->sam.form) == 2) return fail(e, JFGPU_ERR_ARG, "BAM input is taken from host memory only (jfgpu_feed)");
  int rc = begin_feed(e, flags, -1, st);
  if(rc) return rc;
  if((rc = sam_alloc(e))) return rc;
  if(e->part.P) { rc = part_alloc(e); if(rc) return rc; }
  const bool end = flags & JFGPU_FILE_END;
  cudaEventRecord(e->ev_t0, st);
  if(device) rc = sam_feed_device(e, (const uint8_t*)data, n, end, st);
  else if(e->sam.form == 2) rc = bam_feed_host(e, (const char*)data, n, end);
  else rc = sam_feed_host(e, (const char*)data, n, end);
  if(rc) return rc;
  cudaEventRecord(e->ev_t1, st);
  CUDA_OK(e, cudaStreamSynchronize(st));
  { float ms = 0; cudaEventElapsedTime(&ms, e->ev_t0, e->ev_t1); e->count_ms += ms; }
  resolve_kernel_events(e);
  e->bytes_fed += n;
  if(e->tab.slots.p) { rc = check_after_batches(e); if(rc) return rc; }
  return end_feed(e, flags, st);
}

// The transcode of a SAM or BAM file without counting: sam_feed's walk, with sam_run appending every batch's FASTQ to the
// caller's buffer.  The file's carry lives in sam_staged between calls.
static int sam_stage_run(jfgpu_engine* e, const void* data, size_t n, uint32_t flags, bool device, cudaStream_t st) {
  jfgpu_engine::SamState& s = e->sam;
  const uint32_t form = flags & JFGPU_FORMAT_BAM ? 2 : flags & JFGPU_FORMAT_SAM ? 1 : 0;
  if(flags & TEXT_FLAGS) return fail(e, JFGPU_ERR_ARG, "jfgpu_sam_stage takes SAM or BAM input only");
  if((flags & SAM_FLAGS) == SAM_FLAGS) return fail(e, JFGPU_ERR_ARG, "JFGPU_FORMAT_SAM and JFGPU_FORMAT_BAM exclude each other");
  if(flags & JFGPU_FILE_BEGIN) {
    if(!form) return fail(e, JFGPU_ERR_ARG, "jfgpu_sam_stage: JFGPU_FILE_BEGIN needs JFGPU_FORMAT_SAM or JFGPU_FORMAT_BAM");
    sam_begin(s, form);
  } else if(!s.form) {
    return fail(e, JFGPU_ERR_STATE, "jfgpu_sam_stage: no SAM or BAM file is being staged (JFGPU_FILE_BEGIN)");
  } else if(form && form != s.form) {
    return fail(e, JFGPU_ERR_ARG, "the format flag differs from the one the file began with");
  }
  if(device && s.form == 2) return fail(e, JFGPU_ERR_ARG, "BAM input is taken from host memory only");
  int rc = sam_alloc(e);
  if(rc) return rc;
  const bool end = flags & JFGPU_FILE_END;
  if(device) rc = sam_feed_device(e, (const uint8_t*)data, n, end, st);
  else if(s.form == 2) rc = bam_feed_host(e, (const char*)data, n, end);
  else rc = sam_feed_host(e, (const char*)data, n, end);
  if(!rc) CUDA_OK(e, cudaStreamSynchronize(device ? st : e->cs));
  if(rc || end) s.form = 0;                 // (a failed file is not continued)
  return rc;
}

int jfgpu_sam_stage(jfgpu_handle e, const void* bytes, size_t n, uint32_t flags, int on_device, void* dev_out, size_t out_cap,
                    size_t* out_len, void* stream) {
  if(!e || (n && !bytes) || !dev_out || !out_len) return JFGPU_ERR_ARG;
  *out_len = 0;
  cudaSetDevice(e->device);
  cudaStream_t st = stream ? (cudaStream_t)stream : e->cs;
  // host input runs on the engine's streams: the work the caller has queued on `stream` (e.g. on dev_out) comes first
  if(!on_device && stream) CUDA_OK(e, cudaStreamSynchronize(st));
  std::swap(e->sam, e->sam_staged);
  e->stage_out = (uint8_t*)dev_out; e->stage_out_cap = out_cap; e->stage_out_len = 0;
  const int rc = sam_stage_run(e, bytes, n, flags, on_device != 0, st);
  *out_len = e->stage_out_len;
  e->stage_out = nullptr; e->stage_out_cap = e->stage_out_len = 0;
  std::swap(e->sam, e->sam_staged);
  return rc;
}

int jfgpu_feed_device(jfgpu_handle e, const void* dev_bytes, size_t n, uint32_t flags, void* stream) {
  if(!e) return JFGPU_ERR_ARG;
  if(((uintptr_t)dev_bytes & 15) != 0) return fail(e, JFGPU_ERR_ARG, "device text must be 16-byte aligned");
  cudaSetDevice(e->device);
  cudaStream_t st = stream ? (cudaStream_t)stream : e->cs;
  if((flags & SAM_FLAGS) || (e->sam.form && !(flags & JFGPU_FILE_BEGIN))) return sam_feed(e, dev_bytes, n, flags, true, st);
  int rc = begin_device_feed(e, flags, dev_bytes, n, st);
  if(rc) return rc;
  const uint8_t* p = (const uint8_t*)dev_bytes;
  if(e->part.P) { rc = part_alloc(e); if(rc) return rc; }
  cudaEventRecord(e->ev_t0, st);
  for(size_t off = 0; off < n; ) {
    size_t len = std::min(e->part.P ? std::max<size_t>(e->batch_bytes, (size_t)512 << 20) : e->batch_bytes, n - off);
    len = part_cap_len(e, len);
    rc = run_batch(e, p + off, len, n - off, st, K1_COUNT, off);
    if(rc) return rc;
    off += len;
    if((e->p.allow_regrow || e->spill_fn) && !e->part.P && e->tab.slots.p) {          // the failure list only holds two batches
      if(st != e->cs) CUDA_OK(e, cudaStreamSynchronize(st));
      rc = check_after_batches(e);
      if(rc) return rc;
    }
  }
  cudaEventRecord(e->ev_t1, st);
  CUDA_OK(e, cudaStreamSynchronize(st));
  float ms = 0; cudaEventElapsedTime(&ms, e->ev_t0, e->ev_t1); e->count_ms += ms;
  resolve_kernel_events(e);
  e->bytes_fed += n;
  return end_feed(e, flags, st);
}

// length of the longest prefix of [p, p+len) that ends right behind the newline closing a 4-line record, given the number
// of lines (mod 4) in front of p; 0 when there is none.  *lines_out = lines (mod 4) at that point.
static size_t fastq_record_prefix(const char* p, size_t len, uint32_t lines_mod4, uint32_t* lines_out) {
  size_t best = 0; uint32_t lines = lines_mod4, best_lines = lines_mod4;
  const char* q = p; const char* end = p + len;
  while(q < end) {
    const char* nl = (const char*)memchr(q, '\n', (size_t)(end - q));
    if(!nl) break;
    lines = (lines + 1) & 3u;
    q = nl + 1;
    if(lines == 0) { best = (size_t)(q - p); best_lines = 0; }
  }
  *lines_out = best_lines;
  return best;
}

// Length of the next batch of host text at `off`, at most `cap` bytes: it ends in front of a '\r' run that would end it
// (the device looks ahead to see where a run ends; when the run fills all but the first byte, run_staged gives it the byte
// that ends the run), and with `qfastq` (-Q on FASTQ) only behind a complete record (e->q_lines follows).
static int next_batch_len(jfgpu_engine* e, const char* bytes, size_t off, size_t n, size_t cap, bool qfastq, size_t* out) {
  size_t len = cap;
  if(off + len < n) { size_t l2 = len; while(l2 > 1 && bytes[off + l2 - 1] == '\r') --l2; if(l2 > 1) len = l2; }
  if(qfastq && off + len < n) {
    uint32_t l2 = 0;
    const size_t whole = fastq_record_prefix(bytes + off, len, e->q_lines, &l2);
    if(whole == 0) return fail(e, JFGPU_ERR_FORMAT, "Invalid fastq file: a record is larger than the staging buffer (or has more than 4 lines)");
    len = whole; e->q_lines = l2;
  }
  *out = len;
  return JFGPU_OK;
}

int jfgpu_feed(jfgpu_handle e, const char* bytes, size_t n, uint32_t flags) {
  if(!e) return JFGPU_ERR_ARG;
  cudaSetDevice(e->device);
  if((flags & SAM_FLAGS) || (e->sam.form && !(flags & JFGPU_FILE_BEGIN))) return sam_feed(e, bytes, n, flags, false, e->cs);
  int rc = begin_feed(e, flags, n ? (unsigned char)bytes[0] : (e->q_tail.empty() ? -1 : (unsigned char)e->q_tail[0]), e->cs);
  if(rc) return rc;
  if(flags & JFGPU_FILE_BEGIN) { e->q_lines = 0; e->q_tail.clear(); }
  const bool qfastq = eff_min_qual(e) != 0 && e->format == 1;
  std::string joined;                         // (-Q on FASTQ: the incomplete record of the previous feed comes first)
  if(qfastq && !e->q_tail.empty()) {
    joined.swap(e->q_tail);
    joined.append(bytes, n);
    bytes = joined.data(); n = joined.size();
  }
  if(qfastq && !(flags & JFGPU_FILE_END)) {   // keep the incomplete last record for the next feed
    uint32_t l2 = 0;
    const size_t whole = fastq_record_prefix(bytes, n, e->q_lines, &l2);
    e->q_tail.assign(bytes + whole, n - whole);
    n = whole;
  }
  for(int i = 0; i < 2; ++i) if(!e->stage[i].p) CUDA_OK(e, e->stage[i].alloc(e->batch_bytes + 64));
  if(e->part.P) { rc = part_alloc(e); if(rc) return rc; }
  cudaEventRecord(e->ev_t0, e->cs);
  size_t off = 0;
  while(off < n) {
    size_t len = 0;
    rc = next_batch_len(e, bytes, off, n, part_cap_len(e, std::min(e->batch_bytes, n - off)), qfastq, &len);
    if(rc) return rc;
    // the previous batch that used this staging buffer must be done before it is overwritten
    CUDA_OK(e, cudaEventSynchronize(e->ev_done[e->stage_cur]));
    if((e->p.allow_regrow || e->spill_fn) && e->tab.slots.p) {
      // peek at the live failure counter without draining the compute stream
      CUDA_OK(e, cudaMemcpyAsync(e->h_stats + STAT_FAILED, e->stats.as<unsigned long long>() + STAT_FAILED, 8, cudaMemcpyDeviceToHost, e->hs));
      CUDA_OK(e, cudaStreamSynchronize(e->hs));
      if(e->h_stats[STAT_FAILED]) { rc = check_after_batches(e); if(rc) return rc; }
    }
    rc = run_staged(e, bytes, off, len, n, K1_COUNT);
    if(rc) return rc;
    off += len;
  }
  if(qfastq && !(flags & JFGPU_FILE_END)) e->q_lines = 0;       // (the feed was cut behind a complete record)
  cudaEventRecord(e->ev_t1, e->cs);
  e->bytes_fed += n;
  CUDA_OK(e, cudaStreamSynchronize(e->cs));
  { float ms = 0; cudaEventElapsedTime(&ms, e->ev_t0, e->ev_t1); e->count_ms += ms; }
  resolve_kernel_events(e);
  if(e->tab.slots.p) { rc = check_after_batches(e); if(rc) return rc; }
  return end_feed(e, flags, e->cs);
}

// ---- jfgpu_seam: the ordered extraction of a query (K1 MODE 3) over text whose k-mers are not wanted, for the parser state
// and the last symbols it leaves in the carry.  The k-mers go to scratch nobody reads; no table, bucket or filter is touched.
constexpr size_t SEAM_BATCH = (size_t)1 << 20;          // text per launch (the scratch holds the k-mers of that much)

static int seam_begin(jfgpu_engine* e, uint32_t flags, cudaStream_t st, unsigned long long* fmt_err0) {
  if(e->p.min_qual) return fail(e, JFGPU_ERR_ARG, "jfgpu_seam: an engine with min_qual (-Q) reads '\\r' by other rules");
  if(flags & (SAM_FLAGS | JFGPU_FILE_END)) return fail(e, JFGPU_ERR_ARG, "jfgpu_seam takes neither JFGPU_FILE_END nor SAM or BAM input");
  if(e->sam.form && !(flags & JFGPU_FILE_BEGIN)) return fail(e, JFGPU_ERR_ARG, "jfgpu_seam cannot continue a SAM or BAM file");
  if(!e->seam_keys.p) {
    const uint64_t TILE = 512 * 32 - HALO, tiles = (SEAM_BATCH + TILE - 1) / TILE;
    if(make_all(need(e->seam_keys, tiles * TILE * 8 * e->kw), need(e->seam_cnt, tiles * 4)) != cudaSuccess)
      return fail(e, JFGPU_ERR_NOMEM, "allocation of the seam scratch failed");
  }
  CUDA_OK(e, cudaStreamSynchronize(st));
  const int rc = read_stats(e);
  *fmt_err0 = e->h_stats[STAT_FORMAT_ERR];
  return rc;
}

// a FASTQ record the device parser cannot read counts as a format error of the counted text: the seam reports it itself
static int seam_end(jfgpu_engine* e, int rc, cudaStream_t st, unsigned long long fmt_err0) {
  e->seaming = false;
  if(rc) return rc;
  CUDA_OK(e, cudaStreamSynchronize(st));
  rc = read_stats(e);
  if(rc) return rc;
  if(e->h_stats[STAT_FORMAT_ERR] != fmt_err0) {
    CUDA_OK(e, cudaMemcpyAsync(e->stats.as<unsigned long long>() + STAT_FORMAT_ERR, &fmt_err0, 8, cudaMemcpyHostToDevice, e->cs));
    CUDA_OK(e, cudaStreamSynchronize(e->cs));
    e->h_stats[STAT_FORMAT_ERR] = fmt_err0;
    end_feed(e, JFGPU_FILE_END, e->cs);
    return fail(e, JFGPU_ERR_FORMAT, "Invalid fastq sequence (the device parser reads 4-line FASTQ records: '@' header, sequence, '+', qualities)");
  }
  return JFGPU_OK;
}

int jfgpu_seam(jfgpu_handle e, const void* dev_bytes, size_t n, uint32_t flags, void* stream) {
  if(!e || (n && !dev_bytes)) return JFGPU_ERR_ARG;
  if(((uintptr_t)dev_bytes & 15) != 0) return fail(e, JFGPU_ERR_ARG, "device text must be 16-byte aligned");
  cudaSetDevice(e->device);
  cudaStream_t st = stream ? (cudaStream_t)stream : e->cs;
  unsigned long long fmt_err0 = 0;
  int rc = seam_begin(e, flags, st, &fmt_err0);
  if(!rc) rc = begin_device_feed(e, flags, dev_bytes, n, st);
  if(rc) return rc;
  e->seaming = true;
  const uint8_t* p = (const uint8_t*)dev_bytes;
  for(size_t off = 0; off < n && !rc; ) {
    const size_t len = std::min(SEAM_BATCH, n - off);
    rc = run_batch(e, p + off, len, n - off, st, K1_QUERY, off);
    off += len;
  }
  return seam_end(e, rc, st, fmt_err0);
}

int jfgpu_seam_host(jfgpu_handle e, const char* bytes, size_t n, uint32_t flags) {
  if(!e || (n && !bytes)) return JFGPU_ERR_ARG;
  cudaSetDevice(e->device);
  unsigned long long fmt_err0 = 0;
  int rc = seam_begin(e, flags, e->cs, &fmt_err0);
  if(!rc) rc = begin_feed(e, flags, n ? (unsigned char)bytes[0] : -1, e->cs);
  if(rc) return rc;
  for(int i = 0; i < 2; ++i) if(!e->stage[i].p) CUDA_OK(e, e->stage[i].alloc(e->batch_bytes + 64));
  e->seaming = true;
  for(size_t off = 0; off < n && !rc; ) {
    size_t len = 0;
    rc = next_batch_len(e, bytes, off, n, std::min(std::min(SEAM_BATCH, e->batch_bytes), n - off), false, &len);
    if(rc) break;
    // the previous batch that used this staging buffer must be done before it is overwritten
    CUDA_OK(e, cudaEventSynchronize(e->ev_done[e->stage_cur]));
    rc = run_staged(e, bytes, off, len, n, K1_QUERY);
    off += len;
  }
  return seam_end(e, rc, e->cs, fmt_err0);
}

int jfgpu_count_newlines(jfgpu_handle e, const void* dev_bytes, size_t n, uint64_t* dev_count, void* stream) {
  if(!e || (n && (!dev_bytes || !dev_count))) return JFGPU_ERR_ARG;
  cudaSetDevice(e->device);
  cudaStream_t st = stream ? (cudaStream_t)stream : e->cs;
  g_launches.fetch_add(jfnl::count_newlines((const uint8_t*)dev_bytes, n, (unsigned long long*)dev_count, e->n_sm, st), std::memory_order_relaxed);
  CUDA_OK(e, cudaGetLastError());
  return JFGPU_OK;
}

int jfgpu_fastq_cuts(jfgpu_handle e, const void* dev_bytes, size_t n, uint32_t lines_mod4, uint64_t target, uint64_t* cuts,
                     size_t cap, size_t* n_cuts, uint32_t* end_lines_mod4, void* stream) {
  if(!e || (n && !dev_bytes) || !n_cuts || (cap && !cuts) || target == 0) return JFGPU_ERR_ARG;
  if(((uintptr_t)dev_bytes & 15) != 0) return fail(e, JFGPU_ERR_ARG, "device text must be 16-byte aligned");
  cudaSetDevice(e->device);
  cudaStream_t st = stream ? (cudaStream_t)stream : e->cs;
  const size_t need_b = jfnl::fastq_cuts_scratch(n, cap);
  if(e->fq_scratch.bytes < need_b && e->fq_scratch.alloc(need_b) != cudaSuccess)
    return fail(e, JFGPU_ERR_NOMEM, "allocation of the FASTQ cut scratch failed");
  g_launches.fetch_add(jfnl::fastq_cuts((const uint8_t*)dev_bytes, n, lines_mod4, target, cap, e->fq_scratch.p, st), std::memory_order_relaxed);
  CUDA_OK(e, cudaGetLastError());
  jfnl::FqResult r;
  CUDA_OK(e, cudaMemcpyAsync(&r, e->fq_scratch.p, sizeof(r), cudaMemcpyDeviceToHost, st));
  if(cap) CUDA_OK(e, cudaMemcpyAsync(cuts, (const uint8_t*)e->fq_scratch.p + sizeof(r), cap * 8, cudaMemcpyDeviceToHost, st));
  CUDA_OK(e, cudaStreamSynchronize(st));
  if(r.status == 1)
    return fail(e, JFGPU_ERR_FORMAT, "Invalid fastq file: the record at byte " + std::to_string(r.fail_at) + " does not end within " +
                std::to_string(target) + " bytes (a record larger than a piece, or one of more than 4 lines)");
  if(r.status == 2) return fail(e, JFGPU_ERR_ARG, "jfgpu_fastq_cuts: more cuts than `cap`");
  *n_cuts = (size_t)r.n_cuts;
  if(end_lines_mod4) *end_lines_mod4 = (uint32_t)r.end_lines;
  return JFGPU_OK;
}

int jfgpu_extract_route(jfgpu_handle e, const void* dev_bytes, size_t n, uint32_t flags, void* dev_keys, uint64_t capacity,
                        uint64_t* dev_counts, void* stream) {
  if(!e) return JFGPU_ERR_ARG;
  if(flags & SAM_FLAGS) return fail(e, JFGPU_ERR_ARG, "jfgpu_extract_route takes no SAM or BAM input");
  if(!e->tab.slots.p) return fail(e, JFGPU_ERR_STATE, "this engine holds a Bloom counter, not a hash table");
  if(((uintptr_t)dev_bytes & 15) != 0) return fail(e, JFGPU_ERR_ARG, "device text must be 16-byte aligned");
  if(e->kw == 4 && ((uintptr_t)dev_keys & 15) != 0) return fail(e, JFGPU_ERR_ARG, "route buckets of four-word keys must be 16-byte aligned");
  cudaSetDevice(e->device);
  cudaStream_t st = stream ? (cudaStream_t)stream : e->cs;
  int rc = begin_device_feed(e, flags, dev_bytes, n, st);
  if(rc) return rc;
  const uint8_t* p = (const uint8_t*)dev_bytes;
  for(size_t off = 0; off < n; ) {
    size_t len = std::min(e->batch_bytes, n - off);
    rc = run_batch(e, p + off, len, n - off, st, K1_ROUTE, off, 0, (uint64_t*)dev_keys, (unsigned long long*)dev_counts, capacity);
    if(rc) return rc;
    off += len;
  }
  e->bytes_fed += n;
  if(stream && !(flags & (JFGPU_FILE_BEGIN | JFGPU_FILE_END))) return JFGPU_OK;   // stream-ordered: the caller synchronises; drops are reported by jfgpu_finish
  CUDA_OK(e, cudaStreamSynchronize(st));
  rc = end_feed(e, flags, st);
  if(rc) return rc;
  rc = read_stats(e);
  if(rc) return rc;
  if(e->h_stats[STAT_ROUTE_DROPPED]) return fail(e, JFGPU_ERR_FULL, "route bucket capacity exceeded");
  return JFGPU_OK;
}

int jfgpu_shard_setup(jfgpu_handle e, const jfgpu_shard_buffers* b) {
  if(!e || !b) return JFGPU_ERR_ARG;
  cudaSetDevice(e->device);
  const uint32_t G = e->p.n_shards;
  ShardState& sh = e->sh;
  sh.on = false;
  // geometry the record exchange covers: one key word, the 32-bit hash tail, 4-byte records of the GLOBAL regions, the
  // receiver's own partition in 4-byte records drained by the window kernels
  const Table& t = e->tab;
  if(e->kw == 4) return fail(e, JFGPU_ERR_ARG, "the record exchange takes mer lengths up to 64 (k > 64 uses the key exchange)");
  if(G < 2 || G > 8 || !t.slots.p || e->kw != 1 || !t.hash_fast || t.n_prow > 6 || t.lsize > 38 || t.slot_bits != 32 || e->bloom.mode != BLOOM_NONE ||
     !e->part.P || e->part.rec_bytes != 4 || e->part.P > RING_P)
    return fail(e, JFGPU_ERR_ARG, "this table geometry is not covered by the record exchange (use the key exchange)");
  uint32_t P = RING_P;
  while(P > G && t.lsize < ceil_log2(P) + 14) P >>= 1;
  const uint32_t sbits = t.lsize - ceil_log2(P);
  if(sbits + t.hb > 32 || P < G || sbits < e->part.region_bits || (P / G) > e->part.P)
    return fail(e, JFGPU_ERR_ARG, "this table geometry is not covered by the record exchange (use the key exchange)");
  if(!b->send_pool && !b->recv_pool) return JFGPU_OK;          // geometry probe only
  if(!b->send_pool || !b->send_dir || !b->recv_pool || !b->recv_dir || b->send_arena_chunks < 2 * (uint64_t)e->n_sm * (P / G) || b->recv_seg_chunks < b->send_arena_chunks)
    return fail(e, JFGPU_ERR_ARG, "exchange buffers too small: an arena must hold the open chunks of every CTA twice over");
  sh.P = P; sh.sbits = sbits; sh.own_regions = P / G; sh.owner_shift = ceil_log2(P / G); sh.split_lg = sbits - e->part.region_bits;
  sh.arena_chunks = b->send_arena_chunks; sh.seg_chunks = b->recv_seg_chunks;
  sh.send_pool = (uint8_t*)b->send_pool; sh.send_dir = (uint2*)b->send_dir; sh.recv_pool = (uint8_t*)b->recv_pool; sh.recv_dir = (uint2*)b->recv_dir;
  if(make_all(need(sh.pool_next[0], ((size_t)G + 2) * 4), need(sh.pool_next[1], ((size_t)G + 2) * 4), need(sh.cta_chunk, (size_t)e->n_sm * RING_P * 4),
              need(sh.cta_fill, (size_t)e->n_sm * RING_P * 4), need(sh.h_counts, 16 * sizeof(unsigned int))) != cudaSuccess)
    return fail(e, JFGPU_ERR_NOMEM, "device allocation failed");
  for(int i = 0; i < 2; ++i) CUDA_OK(e, cudaMemsetAsync(sh.pool_next[i].p, 0, sh.pool_next[i].bytes, e->cs));
  CUDA_OK(e, cudaMemsetAsync(sh.cta_chunk.p, 0xFF, sh.cta_chunk.bytes, e->cs));
  CUDA_OK(e, cudaMemsetAsync(sh.cta_fill.p, 0, sh.cta_fill.bytes, e->cs));
  CUDA_OK(e, cudaStreamSynchronize(e->cs));
  sh.on = true;
  return JFGPU_OK;
}

uint64_t jfgpu_shard_round_bytes(jfgpu_handle e) {
  if(!e || !e->sh.on) return 0;
  // every byte gives at most one record; iid keys spread evenly over the shards, a third of an arena is kept as slack, and
  // every CTA parks one open chunk per region in the arena of its owner
  const ShardState& sh = e->sh;
  const uint64_t open = (uint64_t)e->n_sm * sh.own_regions;
  const uint64_t room = sh.arena_chunks > open ? sh.arena_chunks - open : 0;
  const uint64_t recs = room * (CHUNK_BYTES / 4 - 2 * RING) * 3 / 4;
  const uint64_t bytes = recs * e->p.n_shards;
  return bytes & ~(uint64_t)0xFFFFF;
}

int jfgpu_shard_extract(jfgpu_handle e, const void* dev_bytes, size_t n, uint32_t flags, uint32_t bank, void* stream) {
  if(!e) return JFGPU_ERR_ARG;
  if(flags & SAM_FLAGS) return fail(e, JFGPU_ERR_ARG, "the record exchange takes no SAM or BAM input");
  if(!e->sh.on || bank > 1) return fail(e, JFGPU_ERR_STATE, "jfgpu_shard_setup has not been called");
  // the record exchange's send kernels apply no Bloom structure: one attached after jfgpu_shard_setup would be ignored
  if(e->bloom.mode != BLOOM_NONE) return fail(e, JFGPU_ERR_STATE, "the record exchange takes no Bloom filter (use the key exchange)");
  if(((uintptr_t)dev_bytes & 15) != 0) return fail(e, JFGPU_ERR_ARG, "device text must be 16-byte aligned");
  cudaSetDevice(e->device);
  cudaStream_t st = stream ? (cudaStream_t)stream : e->cs;
  int rc = begin_device_feed(e, flags, dev_bytes, n, st);
  if(rc) return rc;
  const uint8_t* p = (const uint8_t*)dev_bytes;
  for(size_t off = 0; off < n; ) {
    const size_t len = std::min<size_t>((size_t)512 << 20, n - off);
    rc = run_batch(e, p + off, len, n - off, st, K1_SEND, off, (int)bank);
    if(rc) return rc;
    off += len;
  }
  e->bytes_fed += n;
  if(flags & JFGPU_FILE_END) { CUDA_OK(e, cudaStreamSynchronize(st)); return end_feed(e, flags, st); }
  return JFGPU_OK;                       // stream-ordered
}

int jfgpu_shard_pack(jfgpu_handle e, uint32_t bank, uint64_t* counts, void* stream) {
  if(!e || !counts) return JFGPU_ERR_ARG;
  if(!e->sh.on || bank > 1) return fail(e, JFGPU_ERR_STATE, "jfgpu_shard_setup has not been called");
  cudaSetDevice(e->device);
  cudaStream_t st = stream ? (cudaStream_t)stream : e->cs;
  const uint32_t G = e->p.n_shards;
  PartDev pd = shard_send_dev(e, (int)bank);
  close_chunks_kernel<<<e->n_sm * 4, 256, 0, st>>>(pd, (uint32_t)e->n_sm); JF_LAUNCHED();
  CUDA_OK(e, cudaMemcpyAsync(e->sh.h_counts, pd.pool_next, G * 4, cudaMemcpyDeviceToHost, st));
  CUDA_OK(e, cudaStreamSynchronize(st));
  for(uint32_t d = 0; d < G; ++d) {
    if(e->sh.h_counts[d] > e->sh.arena_chunks) return fail(e, JFGPU_ERR_FULL, "route bucket capacity exceeded (an arena of the send pool overflowed)");
    counts[d] = e->sh.h_counts[d];
  }
  CUDA_OK(e, cudaMemsetAsync(pd.pool_next, 0, ((size_t)G + 2) * 4, st));    // (the chunks stay where they are until the caller has sent them)
  return JFGPU_OK;
}

// restage_kernel over chunks [first, first + count[s]) of every source s's segment (one launch)
static int restage_chunks(jfgpu_engine* e, const uint64_t* count, uint64_t first, uint32_t self_bank, cudaStream_t st) {
  const uint32_t G = e->p.n_shards;
  PartState& ps = e->part;
  uint64_t total = 0;
  for(uint32_t s = 0; s < G; ++s) total += count[s];
  if(total == 0) return JFGPU_OK;
  // room in the CTAs' arenas of the local pool for the records of the received chunks (chunk j goes to CTA j mod grid)
  const uint64_t per_cta = (total + e->n_sm - 1) / e->n_sm + 1;
  int rc = part_reserve(e, st, chunks_for(ps, per_cta * (CHUNK_BYTES / 4)), "record pool smaller than one exchange round");
  if(rc) return rc;
  rc = table_materialize(e, e->tab, st);      // (restage_kernel inserts the records of a full ring or chunk into the table itself)
  if(rc) return rc;
  RestageArgs ra;
  memset(&ra, 0, sizeof(ra));
  ra.T = table_dev(e, e->tab);
  // (the kernel reads chunk rel of source s at s * seg_chunks + rel: the pools seen from chunk `first` on)
  ra.recv_pool = e->sh.recv_pool + first * CHUNK_BYTES; ra.recv_dir = e->sh.recv_dir + first; ra.n_src = G; ra.seg_chunks = (uint32_t)e->sh.seg_chunks;
  for(uint32_t s = 0; s < G; ++s) ra.count[s] = (uint32_t)count[s];
  ra.first_region = e->p.shard_index * e->sh.own_regions; ra.split_lg = e->sh.split_lg; ra.sbits = e->sh.sbits;
  ra.inv_lut = e->tab.inv_lut.as<uint64_t>(); ra.nbytes = e->nbytes;
  if(self_bank <= 1) {             // this shard's own chunks stay in its arena of that send bank
    const size_t a0 = ((size_t)self_bank * G + e->p.shard_index) * e->sh.arena_chunks + first;
    ra.self_pool = e->sh.send_pool + a0 * CHUNK_BYTES; ra.self_dir = e->sh.send_dir + a0; ra.self_src = e->p.shard_index;
  }
  PartDev pd = part_dev(e);
  const size_t smem = (size_t)RING_P * 8 + (size_t)RING_P * RING * 4;
  cudaFuncSetAttribute(restage_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  const int grid = e->n_sm;
  restage_kernel<1><<<grid, 1024, smem, st>>>(ra, pd); JF_LAUNCHED();
  CUDA_OK(e, cudaGetLastError());
  return JFGPU_OK;
}

int jfgpu_shard_unpack(jfgpu_handle e, const uint64_t* counts, uint32_t self_bank, void* stream) {
  if(!e || !counts) return JFGPU_ERR_ARG;
  if(!e->sh.on) return fail(e, JFGPU_ERR_STATE, "jfgpu_shard_setup has not been called");
  cudaSetDevice(e->device);
  cudaStream_t st = stream ? (cudaStream_t)stream : e->cs;
  const uint32_t G = e->p.n_shards;
  int rc = part_alloc(e);
  if(rc) return rc;
  uint64_t total = 0;
  for(uint32_t s = 0; s < G; ++s) { if(counts[s] > std::max(e->sh.seg_chunks, e->sh.arena_chunks)) return fail(e, JFGPU_ERR_ARG, "more chunks than a receive segment holds"); total += counts[s]; }
  const uint64_t slice = std::max<uint64_t>(1, e->fail_group / (CHUNK_BYTES / 4));      // chunks of at most one failure group
  if(!e->spill_fn || total <= slice) {
    rc = restage_chunks(e, counts, 0, self_bank, st);
    return rc || !e->spill_fn ? rc : spill_if_failed(e, st);
  }
  // a spill hook and more records than one failure group (every one of them may meet a full ring or chunk): one source's
  // chunks at a time, cut into slices
  for(uint32_t s = 0; s < G; ++s)
    for(uint64_t first = 0; first < counts[s]; first += slice) {
      uint64_t one[8] = { 0, 0, 0, 0, 0, 0, 0, 0 };
      one[s] = std::min(slice, counts[s] - first);
      rc = restage_chunks(e, one, first, self_bank, st);
      if(!rc) rc = spill_if_failed(e, st);
      if(rc) return rc;
    }
  return JFGPU_OK;
}

// the keys of jfgpu_insert_keys into the table, or as region records into the pool, on `st`
static int insert_key_slice(jfgpu_engine* e, const void* dev_keys, uint64_t n, cudaStream_t st) {
  int rc = JFGPU_OK;
  // --bf-size on a shard: the prefilter runs here, on the owner, where every occurrence of a key arrives (K1 routes them
  // unfiltered, run_batch).  Its matrices are the same draws as on every other shard, also when this one has routed nothing.
  if(e->bloom.mode == BLOOM_FILTER && !e->bloom.drawn && e->op != JFGPU_OP_PRIME) { rc = bloom_draw(e); if(rc) return rc; }
  const BloomDev bf = e->bloom.mode == BLOOM_FILTER ? bloom_dev(e) : BloomDev();
  const size_t bf_smem = bf.mode ? (size_t)e->nbytes * 256 * 8 * 2 : 0;
  PartState& ps = e->part;
  if(ps.P) {
    // region-by-region mode: turn the keys into records of the pool (K1c); K2 inserts them at the next drain
    rc = part_alloc(e);
    if(rc) return rc;
    const uint64_t per_cta = (n + e->n_sm - 1) / e->n_sm + 1024 * 32;     // keys a CTA of stage_keys_kernel handles at most
    rc = part_reserve(e, st, chunks_for(ps, per_cta), "record pool smaller than one batch of keys");
    if(rc) return rc;
  }
  if(ps.P && bf.mode) {
    PartDev pd = part_dev(e);
    TableDev T = table_dev(e, e->tab);
    const size_t smem = (size_t)e->nbytes * 256 * 8 + PMAX * 8 + bf_smem;
    const int grid = (int)std::min<uint64_t>((n + 1024ull * 32 - 1) / (1024ull * 32), (uint64_t)e->n_sm);
    auto kern = bloom_kernels().stage_keys[e->kw - 1];
    cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    kern<<<grid, 1024, smem, st>>>(T, pd, e->tab.lut.as<uint64_t>(), e->nbytes, (const uint64_t*)dev_keys, n, bf);
    JF_LAUNCHED();
    CUDA_OK(e, cudaGetLastError());
  } else if(bf.mode) {
    rc = table_materialize(e, e->tab, st);
    if(rc) return rc;
    TableDev T = table_dev(e, e->tab);
    const size_t smem = (size_t)e->nbytes * 256 * 8 + bf_smem;
    const int grid = (int)std::min<uint64_t>((n + 255) / 256, (uint64_t)e->n_sm * 8);
    rc = dispatch(e, e->kw, e->tab.slot_bits, [&](auto KW, auto SB) -> int {
      auto kern = bloom_kernels().insert_keys[bloom_insert_index<decltype(KW)::value, decltype(SB)::value>()];
      cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
      kern<<<grid, 256, smem, st>>>(T, e->tab.lut.as<uint64_t>(), e->nbytes, (const uint64_t*)dev_keys, n, bf);
      return JFGPU_OK;
    });
    if(rc) return rc;
    JF_LAUNCHED();
    CUDA_OK(e, cudaGetLastError());
  } else if(ps.P) {
    PartDev pd = part_dev(e);
    TableDev T = table_dev(e, e->tab);
    const size_t smem = (size_t)e->nbytes * 256 * 8 + PMAX * 8;
    const int grid = (int)std::min<uint64_t>((n + 1024ull * 32 - 1) / (1024ull * 32), (uint64_t)e->n_sm);
    if(e->kw == 1) {
      cudaFuncSetAttribute(stage_keys_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
      stage_keys_kernel<1><<<grid, 1024, smem, st>>>(T, pd, e->tab.lut.as<uint64_t>(), e->nbytes, (const uint64_t*)dev_keys, n, nullptr);
    } else {
      cudaFuncSetAttribute(stage_keys_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
      stage_keys_kernel<2><<<grid, 1024, smem, st>>>(T, pd, e->tab.lut.as<uint64_t>(), e->nbytes, (const uint64_t*)dev_keys, n, nullptr);
    }
    JF_LAUNCHED();
    CUDA_OK(e, cudaGetLastError());
  } else {
    rc = insert_keys_into(e, e->tab, (const uint64_t*)dev_keys, nullptr, n, st);
    if(rc) return rc;
  }
  return JFGPU_OK;
}

int jfgpu_insert_keys(jfgpu_handle e, const void* dev_keys, uint64_t n, void* stream) {
  if(!e) return JFGPU_ERR_ARG;
  if(!e->tab.slots.p) return fail(e, JFGPU_ERR_STATE, "this engine holds a Bloom counter, not a hash table");
  cudaSetDevice(e->device);
  cudaStream_t st = stream ? (cudaStream_t)stream : e->cs;
  if(n == 0) return JFGPU_OK;
  if(!stream) cudaEventRecord(e->ev_t0, st);
  // with a spill hook, slices of at most one failure group, each followed by the spill its failed keys call for
  const uint64_t slice = e->spill_fn ? e->fail_group : n;
  for(uint64_t off = 0; off < n; off += slice) {
    const uint64_t m = std::min(slice, n - off);
    int rc = insert_key_slice(e, (const uint64_t*)dev_keys + off * e->kw, m, st);
    if(!rc && e->spill_fn) rc = spill_if_failed(e, st);
    if(rc) return rc;
  }
  if(stream) return JFGPU_OK;          // stream-ordered: the caller synchronises
  cudaEventRecord(e->ev_t1, st);
  CUDA_OK(e, cudaStreamSynchronize(st));
  float ms = 0; cudaEventElapsedTime(&ms, e->ev_t0, e->ev_t1); e->count_ms += ms;
  return JFGPU_OK;
}

int jfgpu_set_op(jfgpu_handle e, uint32_t op) {
  if(!e || op > JFGPU_OP_UPDATE) return JFGPU_ERR_ARG;
  // records staged under the previous operation must reach the table under that operation
  int rc = jfgpu_finish(e, nullptr);
  if(rc) return rc;
  e->op = op;
  return JFGPU_OK;
}

int jfgpu_set_spill(jfgpu_handle e, jfgpu_spill_fn fn, void* ctx) {
  if(!e) return JFGPU_ERR_ARG;
  e->spill_fn = fn; e->spill_ctx = ctx;
  return JFGPU_OK;
}

int jfgpu_clear(jfgpu_handle e) {
  if(!e) return JFGPU_ERR_ARG;
  cudaSetDevice(e->device);
  CUDA_OK(e, cudaStreamSynchronize(e->hs));
  CUDA_OK(e, cudaStreamSynchronize(e->cs));
  resolve_kernel_events(e);
  if(e->tab.slots.p) { int rc = table_zero(e, e->tab, lazy_zero_ok(e)); if(rc) return rc; }
  if(e->bloom.bits.p && e->bloom.mode != BLOOM_CHECK) CUDA_OK(e, cudaMemsetAsync(e->bloom.bits.p, 0, e->bloom.bits.bytes, e->cs));
  CUDA_OK(e, cudaMemsetAsync(e->stats.p, 0, STAT_N * 8, e->cs));
  if(e->part.pool.p) {
    CUDA_OK(e, cudaMemsetAsync(e->part.pool_next.p, 0, e->part.pool_next.bytes, e->cs));
    CUDA_OK(e, cudaMemsetAsync(e->part.spill_n.p, 0, 8, e->cs));
    CUDA_OK(e, cudaMemsetAsync(e->part.cta_chunk.p, 0xFF, e->part.cta_chunk.bytes, e->cs));
    CUDA_OK(e, cudaMemsetAsync(e->part.cta_fill.p, 0, e->part.cta_fill.bytes, e->cs));
    e->part.bound_chunks = e->part.P;
    e->part.pending = false;
  }
  if(e->sh.on) {
    for(int i = 0; i < 2; ++i) CUDA_OK(e, cudaMemsetAsync(e->sh.pool_next[i].p, 0, e->sh.pool_next[i].bytes, e->cs));
    CUDA_OK(e, cudaMemsetAsync(e->sh.cta_chunk.p, 0xFF, e->sh.cta_chunk.bytes, e->cs));
    CUDA_OK(e, cudaMemsetAsync(e->sh.cta_fill.p, 0, e->sh.cta_fill.bytes, e->cs));
  }
  e->bytes_fed = 0; e->count_ms = 0; e->kernel_ms = 0; e->kernel_launches = 0; e->drain_ms = 0; e->win_ms[0] = e->win_ms[1] = e->win_ms[2] = 0;
  e->eff_val_len = e->p.counter_len;
  return reset_carry(e, e->cs);
}

int jfgpu_get_stats(jfgpu_handle e, jfgpu_stats* s) {
  if(!e || !s) return JFGPU_ERR_ARG;
  cudaSetDevice(e->device);
  int rc = read_stats(e);
  if(rc) return rc;
  s->kmers = e->h_stats[STAT_KMERS];
  s->inserted = e->h_stats[STAT_INSERTED];
  s->distinct = e->h_stats[STAT_DISTINCT];
  s->reprobes = e->h_stats[STAT_REPROBES];
  s->overflowed = e->h_stats[STAT_OVERFLOWED];
  s->regrows = e->regrows;
  s->bytes = e->bytes_fed;
  s->seconds_count = e->count_ms * 1e-3;
  resolve_kernel_events(e);
  s->seconds_count_kernel = e->kernel_ms * 1e-3;
  s->count_kernel_launches = e->kernel_launches;
  s->seconds_drain = e->drain_ms * 1e-3;
  s->seconds_win_hist = e->win_ms[0] * 1e-3; s->seconds_win_scatter = e->win_ms[1] * 1e-3; s->seconds_win_insert = e->win_ms[2] * 1e-3;
  return JFGPU_OK;
}

int jfgpu_finish(jfgpu_handle e, jfgpu_stats* s) {
  if(!e) return JFGPU_ERR_ARG;
  cudaSetDevice(e->device);
  CUDA_OK(e, cudaStreamSynchronize(e->hs));
  int rc = part_drain(e, e->cs);
  if(!rc) rc = table_materialize(e, e->tab, e->cs);       // (nothing fed since the table was cleared: no drain ran)
  if(rc) return rc;
  CUDA_OK(e, cudaStreamSynchronize(e->cs));
  CUDA_OK(e, cudaGetLastError());
  rc = e->tab.slots.p ? check_after_batches(e) : read_stats(e);
  if(rc) return rc;
  if(e->h_stats[STAT_FORMAT_ERR]) return fail(e, JFGPU_ERR_FORMAT, "Invalid fastq sequence (the device parser reads 4-line FASTQ records: '@' header, sequence, '+', qualities)");
  if(e->h_stats[STAT_POOL_FULL]) return fail(e, JFGPU_ERR_NOMEM, "internal: k-mer record pool overflow");
  if(e->h_stats[STAT_ROUTE_DROPPED]) return fail(e, JFGPU_ERR_FULL, "route bucket capacity exceeded");
  if(e->tab.slots.p) { rc = direct_index_fixup(e); if(rc) return rc; }
  if(s) return jfgpu_get_stats(e, s);
  return JFGPU_OK;
}

int jfgpu_table_info_get(jfgpu_handle e, jfgpu_table_info* info) {
  if(!e || !info) return JFGPU_ERR_ARG;
  if(!e->tab.slots.p) return fail(e, JFGPU_ERR_STATE, "this engine holds a Bloom counter, not a hash table");
  const Table& t = e->tab;
  info->size = t.size; info->lsize = t.lsize; info->key_len = 2 * e->k; info->val_len = e->eff_val_len;
  info->max_reprobe = t.max_reprobe; info->matrix_r = t.M.r(); info->matrix_c = t.M.c();
  info->matrix_identity = t.M.is_low_identity() ? 1 : 0;
  info->slot_bits = t.slot_bits; info->local_slots = t.local_slots; info->table_bytes = t.bytes();
  e->matrix_cols_host.assign(t.M.c(), 0);
  for(unsigned i = 0; i < t.M.c(); ++i) e->matrix_cols_host[i] = t.M[i];
  info->matrix_columns = t.M.is_identity() ? nullptr : e->matrix_cols_host.data();
  info->reprobes = t.reprobes.data();
  info->part_regions = e->part.P; info->part_rec_bytes = e->part.rec_bytes;
  return JFGPU_OK;
}

int jfgpu_dump(jfgpu_handle e, uint64_t lower, uint64_t upper, uint32_t ocl, jfgpu_sink_fn sink, void* ctx, uint64_t* n_records) {
  if(!e || !sink) return JFGPU_ERR_ARG;
  if(!e->tab.slots.p) return fail(e, JFGPU_ERR_STATE, "this engine holds a Bloom counter, not a hash table");
  if(ocl < 1 || ocl > 8) return fail(e, JFGPU_ERR_ARG, "out_counter_len must be in [1, 8]");
  cudaSetDevice(e->device);
  int rc = e->in_spill ? JFGPU_OK : jfgpu_finish(e, nullptr);      // (from inside the spill hook the table is dumped as it stands)
  if(rc) return rc;
  // Segment by segment, two buffers: while the host hands segment i to the sink, the device sorts and serialises segment
  // i+1 (jf_dump.cuh: no global sort, every tile of 8192 positions is ordered in shared memory) and the copy engine brings
  // it to pinned host memory.
  Table& t = e->tab;
  const unsigned rec = e->nbytes + ocl;
  const uint64_t seg = pick_segment(t);
  const uint64_t cap = seg + t.margin + 8;                    // records of a segment at most
  const uint32_t max_tiles = (uint32_t)((seg + DUMP_TP - 1) / DUMP_TP);
  DevBuf tile_cnt[2], out[2];
  HostBuf<uint8_t> hbuf[2];
  HostBuf<uint32_t> h_total;
  Event ev_emit[2], ev_copy[2];
  const unsigned untimed = cudaEventDisableTiming;
  if(make_all(need(h_total, 2 * sizeof(uint32_t)),
              need(tile_cnt[0], ((size_t)max_tiles + 1) * 4), need(out[0], cap * rec + 16), need(hbuf[0], cap * rec + 16), need(ev_emit[0], untimed), need(ev_copy[0], untimed),
              need(tile_cnt[1], ((size_t)max_tiles + 1) * 4), need(out[1], cap * rec + 16), need(hbuf[1], cap * rec + 16), need(ev_emit[1], untimed), need(ev_copy[1], untimed))
     != cudaSuccess) rc = fail(e, JFGPU_ERR_NOMEM, "allocation of the dump buffers failed");
  const size_t smem = (size_t)e->nbytes * 256 * 8 + ((size_t)DUMP_TP + 1) * 4 + (size_t)DUMP_MAXC * 2 + (size_t)DUMP_NTH * rec;
  uint64_t total = 0;
  const uint64_t n_seg = (t.local_size + seg - 1) / seg;
  auto launch = [&](uint64_t si) -> int {            // count, scan, emit of segment si on the compute stream; its total follows
    const int b = (int)(si & 1);
    DumpArgs a;
    memset(&a, 0, sizeof(a));
    a.T = table_dev(e, t);
    a.inv_lut = t.inv_lut.as<uint64_t>(); a.nbytes = e->nbytes; a.ocl = ocl;
    a.seg_lo = si * seg; a.seg_hi = std::min(a.seg_lo + seg, t.local_size);
    a.slots_end = t.local_size + t.margin; a.margin = t.margin;
    a.lower = lower; a.upper = upper;
    a.n_tiles = (uint32_t)((a.seg_hi - a.seg_lo + DUMP_TP - 1) / DUMP_TP);
    a.tile_cnt = tile_cnt[b].as<uint32_t>(); a.out = out[b].as<uint8_t>(); a.out_cap = cap;
    const int grid = (int)std::min<uint64_t>(a.n_tiles, (uint64_t)e->n_sm * 8);
    auto run = [&](auto count_kern, auto kern) -> int {
      count_kern<<<grid, DUMP_NTH, 0, e->cs>>>(a); JF_LAUNCHED();
      dump_scan_kernel<<<1, 1024, 0, e->cs>>>(a.tile_cnt, a.n_tiles); JF_LAUNCHED();
      cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
      kern<<<grid, DUMP_NTH, smem, e->cs>>>(a); JF_LAUNCHED();
      CUDA_OK(e, cudaMemcpyAsync(h_total + b, a.tile_cnt + a.n_tiles, 4, cudaMemcpyDeviceToHost, e->cs));
      CUDA_OK(e, cudaEventRecord(ev_emit[b], e->cs));
      return JFGPU_OK;
    };
    if(e->kw == 4) return run(wide_kernels().dump_count, wide_kernels().dump_emit);
    return dispatch(e, e->kw, t.slot_bits, [&](auto KW, auto SB) -> int {
      constexpr int kw = decltype(KW)::value, sb = decltype(SB)::value;
      return run(dump_count_kernel<sb>, dump_emit_kernel<kw, sb>);
    });
  };
  uint64_t n_in_buf[2] = { 0, 0 };
  if(!rc && n_seg) rc = launch(0);
  for(uint64_t si = 0; si < n_seg && !rc; ++si) {
    const int b = (int)(si & 1);
    // the segment's size, then its bytes on the copy stream
    cudaError_t c = cudaEventSynchronize(ev_emit[b]);
    if(c != cudaSuccess) { rc = fail(e, JFGPU_ERR_CUDA, std::string("dump: ") + cudaGetErrorString(c)); break; }
    n_in_buf[b] = h_total[b];
    if(n_in_buf[b] > cap) { rc = fail(e, JFGPU_ERR_STATE, "internal: segment overflow in dump"); break; }
    if(n_in_buf[b]) cudaMemcpyAsync(hbuf[b], out[b].p, n_in_buf[b] * rec, cudaMemcpyDeviceToHost, e->hs);
    cudaEventRecord(ev_copy[b], e->hs);
    // the next segment is produced while this one is copied and written (its buffers were released two rounds ago)
    if(si + 1 < n_seg) { rc = launch(si + 1); if(rc) break; }
    c = cudaEventSynchronize(ev_copy[b]);
    if(c != cudaSuccess) { rc = fail(e, JFGPU_ERR_CUDA, std::string("dump: ") + cudaGetErrorString(c)); break; }
    if(n_in_buf[b] && sink(ctx, hbuf[b], n_in_buf[b] * rec) != 0) { rc = fail(e, JFGPU_ERR_SINK, "dump sink failed"); break; }
    total += n_in_buf[b];
  }
  cudaStreamSynchronize(e->cs); cudaStreamSynchronize(e->hs);      // (before the buffers go)
  if(n_records) *n_records = total;
  return rc;
}

int jfgpu_lookup(jfgpu_handle e, const uint64_t* keys, size_t n, uint64_t* vals) {
  if(!e || (n && (!keys || !vals))) return JFGPU_ERR_ARG;
  if(!e->tab.slots.p) return fail(e, JFGPU_ERR_STATE, "this engine holds a Bloom counter, not a hash table");
  if(n == 0) return JFGPU_OK;
  cudaSetDevice(e->device);
  { int rc0 = jfgpu_finish(e, nullptr); if(rc0) return rc0; }
  DevBuf dk, dv;
  CUDA_OK(e, dk.alloc(n * 8 * e->kw));
  CUDA_OK(e, dv.alloc(n * 8));
  CUDA_OK(e, cudaMemcpyAsync(dk.p, keys, n * 8 * e->kw, cudaMemcpyHostToDevice, e->cs));
  TableDev T = table_dev(e, e->tab);
  const size_t smem = (size_t)e->nbytes * 256 * 8;
  const int grid = (int)std::min<uint64_t>((n + 255) / 256, (uint64_t)e->n_sm * 8);
  auto run = [&](auto kern) -> int {
    cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    kern<<<grid, 256, smem, e->cs>>>(T, e->tab.lut.as<uint64_t>(), e->nbytes, dk.as<uint64_t>(), n, dv.as<uint64_t>(), e->shard_bits);
    return JFGPU_OK;
  };
  int rc = e->kw == 4 ? run(wide_kernels().lookup)
                      : dispatch(e, e->kw, e->tab.slot_bits, [&](auto KW, auto SB) -> int { return run(lookup_kernel<decltype(KW)::value, decltype(SB)::value>); });
  if(!rc) { JF_LAUNCHED();
    cudaError_t c = cudaMemcpyAsync(vals, dv.p, n * 8, cudaMemcpyDeviceToHost, e->cs);
    if(c == cudaSuccess) c = cudaStreamSynchronize(e->cs);
    if(c != cudaSuccess) rc = fail(e, JFGPU_ERR_CUDA, std::string("lookup: ") + cudaGetErrorString(c));
  }
  return rc;
}

int jfgpu_device_count(void) {
  int n = 0;
  if(cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
  return n;
}

int jfgpu_load_records(jfgpu_handle e, const void* records, size_t nbytes, uint32_t counter_len) {
  if(!e) return JFGPU_ERR_ARG;
  if(!e->tab.slots.p) return fail(e, JFGPU_ERR_STATE, "this engine holds a Bloom counter, not a hash table");
  if(e->shard_bits) return fail(e, JFGPU_ERR_STATE, "a database is loaded into a whole table, not a shard");
  if(counter_len < 1 || counter_len > 8) return fail(e, JFGPU_ERR_ARG, "counter_len must be in [1, 8]");
  const size_t rec = e->nbytes + counter_len;
  if(nbytes % rec) return fail(e, JFGPU_ERR_ARG, "the bytes are not a whole number of records (" + std::to_string(e->nbytes) + " key bytes + " + std::to_string(counter_len) + " count bytes each)");
  if(nbytes && !records) return JFGPU_ERR_ARG;
  cudaSetDevice(e->device);
  int rc = jfgpu_finish(e, nullptr);            // (text fed before is counted first)
  if(rc || nbytes == 0) return rc;
  const uint64_t n_rec = nbytes / rec;
  // a slice is at most one group of the failure list (regrow re-inserts what found no slot)
  const uint64_t slice = std::min<uint64_t>(std::min<uint64_t>(((uint64_t)64 << 20) / rec, e->fail_group), n_rec);
  HostBuf<uint8_t> h[2];
  DevBuf raw, keys, counts;
  if(make_all(need(raw, slice * rec + 16), need(keys, slice * 8 * e->kw), need(counts, slice * 8), need(h[0], slice * rec), need(h[1], slice * rec)) != cudaSuccess)
    rc = fail(e, JFGPU_ERR_NOMEM, "allocation of the load staging buffers failed");
  ForceCount force_count(e);                    // the records' counts are added, whatever the counter is doing
  const uint8_t* src = (const uint8_t*)records;
  if(!rc) memcpy(h[0], src, slice * rec);
  for(uint64_t i = 0, first = 0; first < n_rec && !rc; ++i, first += slice) {
    const uint64_t m = std::min(slice, n_rec - first);
    const int b = (int)(i & 1);
    cudaError_t c = cudaMemcpyAsync(raw.p, h[b], m * rec, cudaMemcpyHostToDevice, e->cs);
    if(c != cudaSuccess) { rc = fail(e, JFGPU_ERR_CUDA, std::string("load: ") + cudaGetErrorString(c)); break; }
    const int grid = (int)std::min<uint64_t>((m + 255) / 256, (uint64_t)e->n_sm * 8);
    if(e->kw == 1) query_decode_kernel<1><<<grid, 256, 0, e->cs>>>(raw.as<uint8_t>(), m, e->nbytes, counter_len, keys.as<uint64_t>(), counts.as<uint64_t>());
    else if(e->kw == 4) wide_kernels().query_decode<<<grid, 256, 0, e->cs>>>(raw.as<uint8_t>(), m, e->nbytes, counter_len, keys.as<uint64_t>(), counts.as<uint64_t>());
    else query_decode_kernel<2><<<grid, 256, 0, e->cs>>>(raw.as<uint8_t>(), m, e->nbytes, counter_len, keys.as<uint64_t>(), counts.as<uint64_t>());
    JF_LAUNCHED();
    rc = insert_keys_into(e, e->tab, keys.as<uint64_t>(), counts.as<uint64_t>(), m, e->cs);
    if(rc) break;
    // the next slice goes to the other pinned buffer while this one is inserted (the copy out of it was enqueued before)
    if(first + m < n_rec) memcpy(h[b ^ 1], src + (first + m) * rec, std::min(slice, n_rec - first - m) * rec);
    rc = check_after_batches(e);                // (synchronises; a table that is full is doubled, counts and all)
  }
  cudaStreamSynchronize(e->cs);                 // (before the staging buffers go)
  // (a full carry side table is not a lack of memory: a larger table would not get a larger one below 2^26 slots)
  if(rc == JFGPU_ERR_FULL && !e->h_stats[STAT_OVF_FULL]) rc = fail(e, JFGPU_ERR_NOMEM, "the database does not fit in device memory (" + e->err + ")");
  return rc;
}

static int query_impl(jfgpu_engine* e, const char* bytes, size_t n, uint32_t flags, jfgpu_sink_fn sink, void* ctx, uint64_t* n_kmers) {
  int rc = jfgpu_finish(e, nullptr);
  if(rc) return rc;
  const unsigned long long fmt_err0 = e->h_stats[STAT_FORMAT_ERR];
  rc = begin_feed(e, flags, n ? (unsigned char)bytes[0] : -1, e->cs);
  if(rc) return rc;
  // batches of at most 16 MB of text: one line per byte at most, up to k + 22 bytes each
  const uint32_t TILE = 512 * 32 - HALO;
  const size_t qbatch = std::min<size_t>(e->batch_bytes, (size_t)16 << 20);
  const uint64_t max_tiles = (qbatch + TILE - 1) / TILE;
  const size_t PIECE = (size_t)64 << 20;        // bytes handed to the sink at most (whole windows: one window's lines < 1.4 MB)
  if(e->q_tiles_cap < max_tiles) {
    CUDA_OK(e, cudaStreamSynchronize(e->cs));
    e->q_tiles_cap = 0;
    const unsigned untimed = cudaEventDisableTiming;
    for(int i = 0; i < 2; ++i) {
      jfgpu_engine::QueryBufs& q = e->qb[i];
      cudaError_t c = make_all(need(q.keys, max_tiles * TILE * 8 * e->kw), need(q.vals, max_tiles * TILE * 8), need(q.cnt, max_tiles * 4),
                               need(q.off, (max_tiles + 1) * 8), need(q.h_off, (max_tiles + 1) * 8), need(q.h_cnt, max_tiles * 4));
      if(c == cudaSuccess && !q.ev_front) c = make_all(need(q.ev_front, untimed), need(q.ev_fmt, untimed));
      if(c == cudaSuccess && !e->q_host[i]) c = make_all(need(e->q_host[i], PIECE), need(e->ev_qcopy[i], untimed));
      if(c != cudaSuccess) return fail(e, JFGPU_ERR_NOMEM, "allocation of the query buffers failed");
    }
    e->q_tiles_cap = max_tiles;
  }
  for(int i = 0; i < 2; ++i) if(!e->stage[i].p) CUDA_OK(e, e->stage[i].alloc(e->batch_bytes + 64));
  TableDev T = table_dev(e, e->tab);
  const size_t lut_smem = (size_t)e->nbytes * 256 * 8;
  // text -> k-mers in order -> counts -> where every window's lines start (enqueued on the compute stream)
  auto front = [&](int b, size_t off, size_t len) -> int {
    jfgpu_engine::QueryBufs& q = e->qb[b];
    CUDA_OK(e, cudaEventSynchronize(e->ev_done[e->stage_cur]));
    e->q_cur = b;
    int rc2 = run_staged(e, bytes, off, len, n, K1_QUERY);
    if(rc2) return rc2;
    q.n_tiles = (len + TILE - 1) / TILE;
    const int grid = (int)std::min<uint64_t>(q.n_tiles, (uint64_t)e->n_sm * 8);
    auto run = [&](auto kern) -> int {
      cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)lut_smem);
      kern<<<grid, QUERY_NTH, lut_smem, e->cs>>>(T, e->tab.lut.as<uint64_t>(), e->nbytes, q.keys.as<uint64_t>(), q.cnt.as<uint32_t>(), TILE,
                                                  q.n_tiles, e->k, 0, q.vals.as<uint64_t>(), q.off.as<unsigned long long>());
      return JFGPU_OK;
    };
    rc2 = e->kw == 4 ? run(wide_kernels().query_lookup)
                     : dispatch(e, e->kw, e->tab.slot_bits, [&](auto KW, auto SB) -> int { return run(query_lookup_kernel<decltype(KW)::value, decltype(SB)::value>); });
    if(rc2) return rc2;
    JF_LAUNCHED();
    query_scan_kernel<<<1, 1024, 0, e->cs>>>(q.off.as<unsigned long long>(), q.n_tiles); JF_LAUNCHED();
    CUDA_OK(e, cudaGetLastError());
    CUDA_OK(e, cudaMemcpyAsync(q.h_off, q.off.p, (q.n_tiles + 1) * 8, cudaMemcpyDeviceToHost, e->cs));
    CUDA_OK(e, cudaMemcpyAsync(q.h_cnt, q.cnt.p, q.n_tiles * 4, cudaMemcpyDeviceToHost, e->cs));
    CUDA_OK(e, cudaEventRecord(q.ev_front, e->cs));
    return JFGPU_OK;
  };
  uint64_t lines = 0;
  size_t off = 0, len = 0;
  if(n) { rc = next_batch_len(e, bytes, 0, n, std::min(qbatch, n), false, &len); if(!rc) rc = front(0, 0, len); }
  for(int b = 0; off < n && !rc; b ^= 1) {
    jfgpu_engine::QueryBufs& q = e->qb[b];
    CUDA_OK(e, cudaEventSynchronize(q.ev_front));
    const uint64_t total = q.h_off[q.n_tiles];
    if(q.out.bytes < total) CUDA_OK(e, q.out.alloc(total + (total >> 3)));
    if(total) {
      const int grid = (int)std::min<uint64_t>(q.n_tiles, (uint64_t)e->n_sm * 8);
      if(e->kw == 1) query_format_kernel<1><<<grid, QUERY_NTH, 0, e->cs>>>(q.keys.as<uint64_t>(), q.vals.as<uint64_t>(), q.cnt.as<uint32_t>(), TILE, 0, q.n_tiles, q.off.as<unsigned long long>(), e->k, q.out.as<uint8_t>());
      else if(e->kw == 4) wide_kernels().query_format<<<grid, QUERY_NTH, 0, e->cs>>>(q.keys.as<uint64_t>(), q.vals.as<uint64_t>(), q.cnt.as<uint32_t>(), TILE, 0, q.n_tiles, q.off.as<unsigned long long>(), e->k, q.out.as<uint8_t>());
      else query_format_kernel<2><<<grid, QUERY_NTH, 0, e->cs>>>(q.keys.as<uint64_t>(), q.vals.as<uint64_t>(), q.cnt.as<uint32_t>(), TILE, 0, q.n_tiles, q.off.as<unsigned long long>(), e->k, q.out.as<uint8_t>());
      JF_LAUNCHED();
      CUDA_OK(e, cudaGetLastError());
    }
    CUDA_OK(e, cudaEventRecord(q.ev_fmt, e->cs));
    for(uint64_t t = 0; t < q.n_tiles; ++t) lines += q.h_cnt[t];
    // the next batch is extracted and looked up while the lines of this one go out
    off += len;
    if(off < n) {
      rc = next_batch_len(e, bytes, off, n, std::min(qbatch, n - off), false, &len);
      if(!rc) rc = front(b ^ 1, off, len);
      if(rc) break;
    }
    // pieces of whole windows, copied through two pinned buffers: piece j+1 is copied while the sink takes piece j
    std::vector<std::pair<uint64_t, uint64_t>> pieces;          // byte ranges of the batch's output
    for(uint64_t t = 0; t < q.n_tiles; ) {
      uint64_t u = t + 1;
      while(u < q.n_tiles && q.h_off[u + 1] - q.h_off[t] <= PIECE) ++u;
      if(q.h_off[u] > q.h_off[t]) pieces.push_back(std::make_pair(q.h_off[t], q.h_off[u] - q.h_off[t]));
      t = u;
    }
    CUDA_OK(e, cudaStreamWaitEvent(e->hs, q.ev_fmt, 0));
    auto copy = [&](size_t j) -> int {
      CUDA_OK(e, cudaMemcpyAsync(e->q_host[j & 1], q.out.as<uint8_t>() + pieces[j].first, pieces[j].second, cudaMemcpyDeviceToHost, e->hs));
      CUDA_OK(e, cudaEventRecord(e->ev_qcopy[j & 1], e->hs));
      return JFGPU_OK;
    };
    if(!pieces.empty()) rc = copy(0);
    for(size_t j = 0; j < pieces.size() && !rc; ++j) {
      if(j + 1 < pieces.size()) { rc = copy(j + 1); if(rc) break; }
      CUDA_OK(e, cudaEventSynchronize(e->ev_qcopy[j & 1]));
      if(sink(ctx, e->q_host[j & 1], pieces[j].second) != 0) rc = fail(e, JFGPU_ERR_SINK, "query sink failed");
    }
  }
  CUDA_OK(e, cudaStreamSynchronize(e->cs));
  CUDA_OK(e, cudaStreamSynchronize(e->hs));
  if(rc) return rc;
  if(n_kmers) *n_kmers = lines;
  rc = read_stats(e);
  if(rc) return rc;
  if(e->h_stats[STAT_FORMAT_ERR] != fmt_err0) {         // (the counter is put back: the table's own text had no such error)
    CUDA_OK(e, cudaMemcpyAsync(e->stats.as<unsigned long long>() + STAT_FORMAT_ERR, &fmt_err0, 8, cudaMemcpyHostToDevice, e->cs));
    CUDA_OK(e, cudaStreamSynchronize(e->cs));
    e->h_stats[STAT_FORMAT_ERR] = fmt_err0;
    end_feed(e, JFGPU_FILE_END, e->cs);
    return fail(e, JFGPU_ERR_FORMAT, "Invalid fastq sequence (the device parser reads 4-line FASTQ records: '@' header, sequence, '+', qualities)");
  }
  return end_feed(e, flags, e->cs);
}

int jfgpu_query(jfgpu_handle e, const char* bytes, size_t n, uint32_t flags, jfgpu_sink_fn sink, void* ctx, uint64_t* n_kmers) {
  if(!e || !sink || (n && !bytes)) return JFGPU_ERR_ARG;
  if(flags & SAM_FLAGS) return fail(e, JFGPU_ERR_ARG, "a query takes no SAM or BAM input");
  if(n_kmers) *n_kmers = 0;
  if(!e->tab.slots.p) return fail(e, JFGPU_ERR_STATE, "this engine holds a Bloom counter, not a hash table");
  if(e->shard_bits) return fail(e, JFGPU_ERR_STATE, "a query needs the whole table, not a shard");
  cudaSetDevice(e->device);
  e->querying = true;
  const int rc = query_impl(e, bytes, n, flags, sink, ctx, n_kmers);
  e->querying = false;
  return rc;
}

int jfgpu_histogram(jfgpu_handle e, uint64_t* hist, uint32_t n_bins) {
  if(!e || !hist || n_bins == 0) return JFGPU_ERR_ARG;
  if(!e->tab.slots.p) return fail(e, JFGPU_ERR_STATE, "this engine holds a Bloom counter, not a hash table");
  cudaSetDevice(e->device);
  int rc = jfgpu_finish(e, nullptr);
  if(rc) return rc;
  DevBuf dh;
  CUDA_OK(e, dh.alloc((size_t)n_bins * 8));
  CUDA_OK(e, cudaMemsetAsync(dh.p, 0, (size_t)n_bins * 8, e->cs));
  TableDev T = table_dev(e, e->tab);
  const uint64_t ns = e->tab.local_size + e->tab.margin;
  const int grid = (int)std::min<uint64_t>((ns + 255) / 256, (uint64_t)e->n_sm * 16);
  switch(e->tab.slot_bits) {
  case 32:  histogram_kernel<32><<<grid, 256, 0, e->cs>>>(T, ns, dh.as<unsigned long long>(), n_bins); break;
  case 64:  histogram_kernel<64><<<grid, 256, 0, e->cs>>>(T, ns, dh.as<unsigned long long>(), n_bins); break;
  case SB_WIDE: wide_kernels().histogram<<<grid, 256, 0, e->cs>>>(T, ns, dh.as<unsigned long long>(), n_bins); break;
  default:  histogram_kernel<128><<<grid, 256, 0, e->cs>>>(T, ns, dh.as<unsigned long long>(), n_bins); break;
  }
  JF_LAUNCHED();
  cudaError_t c = cudaMemcpyAsync(hist, dh.p, (size_t)n_bins * 8, cudaMemcpyDeviceToHost, e->cs);
  if(c == cudaSuccess) c = cudaStreamSynchronize(e->cs);
  if(c != cudaSuccess) return fail(e, JFGPU_ERR_CUDA, std::string("histogram: ") + cudaGetErrorString(c));
  return JFGPU_OK;
}

int jfgpu_bloom_info_get(jfgpu_handle e, jfgpu_bloom_info* info) {
  if(!e || !info) return JFGPU_ERR_ARG;
  cudaSetDevice(e->device);
  memset(info, 0, sizeof(*info));
  BloomState& b = e->bloom;
  info->mode = b.mode;
  if(b.mode == BLOOM_NONE) return JFGPU_OK;
  if(!b.drawn) { int rc = bloom_draw(e); if(rc) return rc; }
  info->nb_hashes = b.k; info->m = b.m;
  info->nb_bytes = b.mode == BLOOM_FILTER ? b.m / 8 + (b.m % 8 != 0) : b.m / 5 + (b.m % 5 != 0);
  info->matrix_r = 64; info->matrix_c = 2 * e->k;
  info->matrix1 = b.cols1.data(); info->matrix2 = b.cols2.data();
  return JFGPU_OK;
}

int jfgpu_bloom_load(jfgpu_handle e, uint64_t m, uint32_t nb_hashes, const uint64_t* c1, const uint64_t* c2, const void* bytes, size_t nbytes) {
  if(!e || !c1 || !c2 || !bytes) return JFGPU_ERR_ARG;
  cudaSetDevice(e->device);
  if(!e->tab.slots.p) return fail(e, JFGPU_ERR_STATE, "this engine holds a Bloom counter, not a hash table");
  if(e->bloom.mode != BLOOM_NONE) return fail(e, JFGPU_ERR_STATE, "a Bloom filter is already attached to this engine");
  if(m == 0 || nb_hashes == 0) return fail(e, JFGPU_ERR_ARG, "empty Bloom counter");
  if(nbytes < m / 5 + (m % 5 != 0)) return fail(e, JFGPU_ERR_ARG, "Bloom filter file is truncated");
  int rc = jfgpu_finish(e, nullptr);          // text fed so far is counted unfiltered
  if(rc) return rc;
  BloomState& b = e->bloom;
  b.m = m; b.k = nb_hashes;
  b.inv = m == 1 ? ~(uint64_t)0 : (uint64_t)(((unsigned __int128)1 << 64) / m);
  b.n_words = (m + 31) / 32;
  {
    DevBuf raw;                  // (goes at the end of this block, before the hash tables are uploaded)
    const size_t nb = m / 5 + (m % 5 != 0);
    if(make_all(need(b.bits, (size_t)b.n_words * 4 + 16), need(raw, nb + 16)) != cudaSuccess)
      return fail(e, JFGPU_ERR_NOMEM, "Failed to allocate the Bloom counter in device memory");
    CUDA_OK(e, cudaMemcpyAsync(raw.p, bytes, nb, cudaMemcpyHostToDevice, e->cs));
    const int grid = (int)std::min<uint64_t>((b.n_words + 255) / 256, (uint64_t)e->n_sm * 16);
    bloom_unpack_kernel<<<grid, 256, 0, e->cs>>>(raw.as<uint8_t>(), m, b.n_words, b.bits.as<uint32_t>()); JF_LAUNCHED();
    CUDA_OK(e, cudaStreamSynchronize(e->cs));
  }
  b.M1 = jfb::gf2_matrix(64, 2 * e->k, c1); b.M2 = jfb::gf2_matrix(64, 2 * e->k, c2);
  b.mode = BLOOM_CHECK;
  return bloom_upload_matrices(e);
}

int jfgpu_bloom_words(jfgpu_handle e, void** dev_words, uint64_t* n_words) {
  if(!e || !dev_words || !n_words) return JFGPU_ERR_ARG;
  cudaSetDevice(e->device);
  const BloomState& b = e->bloom;
  if(b.mode != BLOOM_COUNT) return fail(e, JFGPU_ERR_STATE, "no Bloom counter has been built by this engine");
  int rc = jfgpu_finish(e, nullptr);           // (the words are complete for the caller's streams)
  if(rc) return rc;
  *dev_words = b.bits.p; *n_words = b.n_words;
  return JFGPU_OK;
}

int jfgpu_bloom_fold(jfgpu_handle e, const void* dev_words, uint64_t first_word, uint64_t n_words, void* stream) {
  if(!e || (!dev_words && n_words)) return JFGPU_ERR_ARG;
  cudaSetDevice(e->device);
  const BloomState& b = e->bloom;
  if(b.mode != BLOOM_COUNT) return fail(e, JFGPU_ERR_STATE, "no Bloom counter has been built by this engine");
  if(first_word > b.n_words || n_words > b.n_words - first_word) return fail(e, JFGPU_ERR_ARG, "word range outside the Bloom counter");
  if(n_words == 0) return JFGPU_OK;
  cudaStream_t st = stream ? (cudaStream_t)stream : e->cs;
  const int grid = (int)std::min<uint64_t>((n_words + 255) / 256, (uint64_t)e->n_sm * 16);
  bloom_kernels().fold<<<grid, 256, 0, st>>>(b.bits.as<uint32_t>() + first_word, (const uint32_t*)dev_words, n_words); JF_LAUNCHED();
  CUDA_OK(e, cudaGetLastError());
  return JFGPU_OK;
}

int jfgpu_bloom_dump_range(jfgpu_handle e, uint64_t first_byte, uint64_t n_bytes, jfgpu_sink_fn sink, void* ctx) {
  if(!e || !sink) return JFGPU_ERR_ARG;
  cudaSetDevice(e->device);
  BloomState& b = e->bloom;
  if(b.mode != BLOOM_COUNT) return fail(e, JFGPU_ERR_STATE, "no Bloom counter has been built by this engine");
  const uint64_t nb = b.m / 5 + (b.m % 5 != 0);
  if(first_byte % 16 != 0) return fail(e, JFGPU_ERR_ARG, "the first byte of a Bloom counter range must be a multiple of 16");
  if(first_byte > nb || n_bytes > nb - first_byte) return fail(e, JFGPU_ERR_ARG, "byte range outside the Bloom counter");
  int rc = jfgpu_finish(e, nullptr);
  if(rc) return rc;
  const uint64_t piece = (uint64_t)64 << 20;
  DevBuf out; HostBuf<uint8_t> hbuf;
  if(make_all(need(out, piece), need(hbuf, piece)) != cudaSuccess) return fail(e, JFGPU_ERR_NOMEM, "allocation of the Bloom counter staging buffers failed");
  const uint64_t end = first_byte + n_bytes;
  for(uint64_t off = first_byte; off < end && !rc; off += piece) {
    const uint64_t len = std::min(piece, end - off);
    const int grid = (int)std::min<uint64_t>((len + 255) / 256, (uint64_t)e->n_sm * 16);
    // positions 5*off .. : the kernel takes the bit array shifted by whole words (5*off*2 bits; piece is a multiple of 16 bytes)
    bloom_pack_kernel<<<grid, 256, 0, e->cs>>>(b.bits.as<uint32_t>() + (5 * off) / 16, b.m - 5 * off, len, out.as<uint8_t>()); JF_LAUNCHED();
    cudaError_t c = cudaMemcpyAsync(hbuf, out.p, len, cudaMemcpyDeviceToHost, e->cs);
    if(c == cudaSuccess) c = cudaStreamSynchronize(e->cs);
    if(c != cudaSuccess) { rc = fail(e, JFGPU_ERR_CUDA, std::string("bloom dump: ") + cudaGetErrorString(c)); break; }
    if(sink(ctx, hbuf, len) != 0) rc = fail(e, JFGPU_ERR_SINK, "dump sink failed");
  }
  return rc;
}

int jfgpu_bloom_dump(jfgpu_handle e, jfgpu_sink_fn sink, void* ctx) {
  if(!e || !sink) return JFGPU_ERR_ARG;
  if(e->bloom.mode != BLOOM_COUNT) return fail(e, JFGPU_ERR_STATE, "no Bloom counter has been built by this engine");
  return jfgpu_bloom_dump_range(e, 0, e->bloom.m / 5 + (e->bloom.m % 5 != 0), sink, ctx);
}

uint64_t jfgpu_synth_fasta_bytes(uint64_t n_bases) {
  return SYNTH_HDR + n_bases + (n_bases + SYNTH_LINE - 1) / SYNTH_LINE;
}

int jfgpu_synth_fasta_device(int device, void* dev_out, uint64_t capacity, uint64_t n_bases, uint64_t seed, uint64_t* n_bytes, void* stream) {
  const uint64_t need = jfgpu_synth_fasta_bytes(n_bases);
  if(!dev_out || capacity < need) return JFGPU_ERR_ARG;
  if(cudaSetDevice(device) != cudaSuccess) { cudaGetLastError(); return JFGPU_ERR_CUDA; }
  const int grid = (int)std::min<uint64_t>((need + 255) / 256, (uint64_t)132 * 32);
  synth_fasta_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>((uint8_t*)dev_out, need, n_bases, seed);
  JF_LAUNCHED();
  if(cudaGetLastError() != cudaSuccess) return JFGPU_ERR_CUDA;
  if(n_bytes) *n_bytes = need;
  return JFGPU_OK;
}

}  // extern "C"
