// jf_kernels.cuh -- the sm_90a kernels of the counting pipeline.
//
//   K0a nl_scan_kernel      last '\n' of every tile (two ranges, see tile_state_kernel)
//   K0b tile_state_kernel   parser state at the start of every staged window
//   K1  extract_kernel      (jf_extract.cuh) fused: TMA-staged text window -> word-parallel classification -> packed symbol
//                           streams -> canonical k-mers -> GF(2) hash -> CAS insert (MODE 0), bucket by owning shard
//                           (MODE 1), compact region records appended to per-CTA chunk lists (MODE 2), or the keys
//                           themselves in input order, per window (MODE 3, `query -s`; jf_query.cuh takes it from there)
//   K2  win_* kernels       (jf_window.cuh) region records -> table, one shared-memory window at a time;
//       insert_chunks*      the L2 form of the same for slot widths the window form does not cover
//   K2' insert_keys_kernel  packed keys -> hash -> insert (multi-GPU receive side, regrow, spilled records)
//   K3  collect_kernel      table segment -> (key, count) pairs (regrow);  dump_* kernels (jf_dump.cuh): sorted record bytes
//   K5  lookup / histogram / synth_fasta
#ifndef JF_KERNELS_CUH
#define JF_KERNELS_CUH
#include "jf_device.cuh"

namespace jfk {

// ---------------------------------------------------------------------------------------
// K0a: per tile t (bytes [t*TILE, (t+1)*TILE)), position of the last '\n' in
//      A = [start, start+TILE-HALO) and in B = [start+TILE-HALO, start+TILE); -1 if none.
// ---------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) nl_scan_kernel(const uint8_t* __restrict__ in, uint64_t n, uint64_t n_tiles, uint32_t TILE,
                                                      long long* __restrict__ nlA, long long* __restrict__ nlB,
                                                      uint32_t* __restrict__ cntA, uint32_t* __restrict__ cntB) {
  __shared__ long long sA[8], sB[8];
  __shared__ uint32_t sCA[8], sCB[8];
  for(uint64_t t = blockIdx.x; t < n_tiles; t += gridDim.x) {
    const uint64_t start = t * (uint64_t)TILE;
    const uint64_t end = min(n, start + (uint64_t)TILE);
    const uint64_t split = start + (uint64_t)(TILE - HALO);
    long long a = -1, b = -1;
    uint32_t ca = 0, cb = 0;
    // 16-byte vectors; the tile start is 16-byte aligned
    const uint64_t nvec = (end - start) / 16;
    const uint4* v = reinterpret_cast<const uint4*>(in + start);
    for(uint64_t i = threadIdx.x; i < nvec; i += blockDim.x) {
      uint4 x = v[i];
      uint32_t w[4] = { x.x, x.y, x.z, x.w };
#pragma unroll
      for(int j = 0; j < 4; ++j) {
        uint32_t y = w[j] ^ 0x0A0A0A0Au;
        if(((y - 0x01010101u) & ~y & 0x80808080u) != 0u) {     // some byte of w[j] is '\n'
#pragma unroll
          for(int q = 0; q < 4; ++q) {
            if(((w[j] >> (8 * q)) & 0xFFu) == 0x0Au) {
              long long p = (long long)(start + i * 16 + j * 4 + q);
              if((uint64_t)p < split) { a = max(a, p); ++ca; } else { b = max(b, p); ++cb; }
            }
          }
        }
      }
    }
    for(uint64_t p = start + nvec * 16 + threadIdx.x; p < end; p += blockDim.x) {
      if(in[p] == '\n') { if(p < split) { a = max(a, (long long)p); ++ca; } else { b = max(b, (long long)p); ++cb; } }
    }
#pragma unroll
    for(int o = 16; o; o >>= 1) {
      a = max(a, __shfl_xor_sync(0xffffffffu, a, o));
      b = max(b, __shfl_xor_sync(0xffffffffu, b, o));
      ca += __shfl_xor_sync(0xffffffffu, ca, o);
      cb += __shfl_xor_sync(0xffffffffu, cb, o);
    }
    if((threadIdx.x & 31) == 0) { sA[threadIdx.x >> 5] = a; sB[threadIdx.x >> 5] = b; sCA[threadIdx.x >> 5] = ca; sCB[threadIdx.x >> 5] = cb; }
    __syncthreads();
    if(threadIdx.x == 0) {
      for(int i = 1; i < (int)(blockDim.x >> 5); ++i) { a = max(a, sA[i]); b = max(b, sB[i]); ca += sCA[i]; cb += sCB[i]; }
      nlA[t] = a; nlB[t] = b; cntA[t] = ca; cntB[t] = cb;
    }
    __syncthreads();
  }
}

// state after the bytes [from, to) when entering them at a line start / with state s0
// (keep_cr: -Q semantics, std::getline keeps a leading '\r': the line is then a sequence line)
__device__ __forceinline__ uint32_t line_start_state(const uint8_t* in, uint64_t from, uint64_t to, uint32_t s0, bool keep_cr = false) {
  if(s0 != ST_L) return s0;
  uint64_t p = from;
  while(!keep_cr && p < to && in[p] == '\r') ++p;
  if(p >= to) return ST_L;
  return in[p] == '>' ? ST_H : ST_S;
}

// ---------------------------------------------------------------------------------------
// K0b: window t starts at h_t = t*TILE - HALO.  Its entry state depends on the last '\n'
//      before h_t:  max(nlA[t-1], max_{u<t-1} max(nlA[u], nlB[u])).  One CTA, chunked scan:
//      the thread that owns tile u produces the state of window u+1.
// ---------------------------------------------------------------------------------------
__global__ void __launch_bounds__(1024) tile_state_kernel(const uint8_t* __restrict__ in, uint64_t n_tiles, uint32_t TILE,
                                                          const long long* __restrict__ nlA, const long long* __restrict__ nlB,
                                                          const Carry* __restrict__ carry_in, uint8_t* __restrict__ tile_state, uint32_t keep_cr) {
  __shared__ long long part[1024];
  const uint64_t per = (n_tiles + blockDim.x - 1) / blockDim.x;
  const uint64_t lo = min(n_tiles, per * threadIdx.x), hi = min(n_tiles, lo + per);
  long long m = -1;
  for(uint64_t u = lo; u < hi; ++u) m = max(m, max(nlA[u], nlB[u]));
  part[threadIdx.x] = m;
  __syncthreads();
  if(threadIdx.x == 0) {               // exclusive running max over the partials
    long long run = -1;
    for(int i = 0; i < (int)blockDim.x; ++i) { long long x = part[i]; part[i] = run; run = max(run, x); }
  }
  __syncthreads();
  long long mu = part[threadIdx.x];    // last newline in tiles < u   (u = lo initially)
  const uint32_t cstate = carry_in->state;
  if(threadIdx.x == 0 && n_tiles) tile_state[0] = (uint8_t)cstate;
  for(uint64_t u = lo; u < hi; ++u) {
    if(u + 1 < n_tiles) {
      const long long before = max(mu, nlA[u]);               // last newline before h_{u+1}
      const uint64_t h = (u + 1) * (uint64_t)TILE - HALO;
      tile_state[u + 1] = (uint8_t)(before >= 0 ? line_start_state(in, (uint64_t)before + 1, h, ST_L, keep_cr != 0)
                                                : line_start_state(in, 0, h, cstate, keep_cr != 0));
    }
    mu = max(mu, max(nlA[u], nlB[u]));
  }
}

// FASTQ: line type at the start of every window = (type at the batch start + newlines before it) mod 4
__global__ void __launch_bounds__(1024) tile_state_fastq_kernel(uint64_t n_tiles, const uint32_t* __restrict__ cntA, const uint32_t* __restrict__ cntB,
                                                                const Carry* __restrict__ carry_in, uint8_t* __restrict__ tile_state) {
  __shared__ uint32_t part[1024];
  const uint64_t per = (n_tiles + blockDim.x - 1) / blockDim.x;
  const uint64_t lo = min(n_tiles, per * threadIdx.x), hi = min(n_tiles, lo + per);
  uint32_t m = 0;
  for(uint64_t u = lo; u < hi; ++u) m += cntA[u] + cntB[u];
  part[threadIdx.x] = m;
  __syncthreads();
  if(threadIdx.x == 0) { uint32_t run = 0; for(int i = 0; i < (int)blockDim.x; ++i) { uint32_t x = part[i]; part[i] = run; run += x; } }
  __syncthreads();
  uint32_t mu = part[threadIdx.x];     // newlines in tiles < u (mod 2^32 is fine: only mod 4 matters)
  const uint32_t ctype = carry_in->state & 3u;
  if(threadIdx.x == 0 && n_tiles) tile_state[0] = (uint8_t)ctype;
  for(uint64_t u = lo; u < hi; ++u) {
    if(u + 1 < n_tiles) tile_state[u + 1] = (uint8_t)((ctype + mu + cntA[u]) & 3u);
    mu += cntA[u] + cntB[u];
  }
}

// ---------------------------------------------------------------------------------------
// parser state machine helpers (semantics: mer_overlap_sequence_parser.hpp:161-185,260-287)
//   state L (line start): '\n','\r' stay; '>' -> H (new record: emits a window reset, the 'N'
//                          of :174-176); anything else -> S and is a sequence character
//   state S (in sequence): '\n' -> L; '\r' dropped when the run of '\r' ends in '\n'/EOF,
//                          otherwise it is a window reset; other bytes: base or reset
//   state H (in header)  : '\n' -> L; everything else ignored
// A transition function over {H,S,L} is packed 2 bits per input state.
// ---------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t fn_const(uint32_t s) { return s | (s << 2) | (s << 4) | (s << 6); }
__device__ __forceinline__ uint32_t fn_apply(uint32_t f, uint32_t s) { return (f >> (2 * s)) & 3u; }
// first f, then g
__device__ __forceinline__ uint32_t fn_compose(uint32_t f, uint32_t g) {
  return fn_apply(g, fn_apply(f, 0)) | (fn_apply(g, fn_apply(f, 1)) << 2) | (fn_apply(g, fn_apply(f, 2)) << 4) |
         (fn_apply(g, fn_apply(f, 3)) << 6);
}
constexpr uint32_t FN_ID = 0u | (1u << 2) | (2u << 4) | (3u << 6);
// FASTQ: the state is the line type 0..3 (header '@', sequence, '+', qualities) of 4-line records;
// a piece of text containing n newlines advances it by n
__device__ __forceinline__ uint32_t fn_rot(uint32_t n) {
  n &= 3u;
  return (n & 3u) | (((1 + n) & 3u) << 2) | (((2 + n) & 3u) << 4) | (((3 + n) & 3u) << 6);
}

// is the '\r' at position p (inside a sequence line) dropped?  True when the run of '\r'
// it belongs to is followed by '\n' or by the end of the file.
__device__ __forceinline__ bool cr_dropped(const uint8_t* in, uint64_t p, uint64_t n) {
  uint64_t q = p + 1;
  while(q < n && in[q] == '\r') ++q;
  return q >= n || in[q] == '\n';
}

struct CountArgs {
  const uint8_t* in;          // batch bytes (16-byte aligned)
  uint64_t       n;           // bytes in the batch
  uint64_t       n_look;      // bytes readable from `in` (>= n): look-ahead for '\r' runs
  uint64_t       n_tiles;
  const uint8_t* tile_state;
  const Carry*   carry_in;
  Carry*         carry_out;
  const uint64_t* lut;        // nb*256 hash table entries (global)
  uint32_t       k;
  uint32_t       canonical;
  uint32_t       nbytes;      // ceil(2k/8)
  uint32_t       mode;        // 0 = insert, 1 = route
  TableDev       T;
  // route mode
  uint64_t*      route_keys;
  unsigned long long* route_counts;
  uint64_t       route_cap;
  uint32_t       shard_bits;
  // fast hash (2k <= 44): four 11-bit-indexed tables of 32-bit entries give the low 32 position bits,
  // the few bits above come from parity rows
  uint32_t       hash_fast;
  uint32_t       n_prow;
  uint32_t       lut_bytes;     // bytes of hash tables to stage in shared memory
  uint32_t       format;        // 0 = FASTA, 1 = FASTQ (4-line records)
  uint32_t       min_qual;      // -Q / --min-quality (0 = off): a base whose quality character is below this one resets the window;
                                // whole_sequence_parser line semantics ('\r' is an ordinary, i.e. resetting, character)
  uint64_t       n_back;        // bytes readable in front of `in` (the line a window starts in may begin there)
  uint64_t       prow[8];
  BloomDev       bloom;         // filter in front of the table (mode BLOOM_NONE: nothing)
  // ordered extraction (MODE 3, `query -s`): the k-mers of window t, in input order, at q_keys[(t*q_tile_cap + i)*KW],
  // i < q_cnt[t]
  uint64_t*      q_keys;
  uint32_t*      q_cnt;
  uint32_t       q_tile_cap;
};

// the Bloom counter as `jellyfish bc` writes it (bloom_counter2.hpp:34-36: five base-3 digits per byte) from the two-bit form
__global__ void __launch_bounds__(256) bloom_pack_kernel(const uint32_t* __restrict__ bits, uint64_t m, uint64_t n_bytes, uint8_t* __restrict__ out) {
  for(uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; j < n_bytes; j += (uint64_t)gridDim.x * blockDim.x) {
    uint32_t v = 0, pw = 1;
    for(uint32_t i = 0; i < 5; ++i, pw *= 3) {
      const uint64_t pos = 5 * j + i;
      if(pos < m) { const uint32_t f = (bits[pos >> 4] >> ((pos & 15u) * 2u)) & 3u; v += ((f & 1u) + (f >> 1)) * pw; }
    }
    out[j] = (uint8_t)v;
  }
}
// ... and the "digit is 2" bitmap of a loaded counter (count --bc)
__global__ void __launch_bounds__(256) bloom_unpack_kernel(const uint8_t* __restrict__ bytes, uint64_t m, uint64_t n_words, uint32_t* __restrict__ out) {
  for(uint64_t w = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; w < n_words; w += (uint64_t)gridDim.x * blockDim.x) {
    uint32_t x = 0;
    for(uint32_t b = 0; b < 32; ++b) {
      const uint64_t pos = 32 * w + b;
      if(pos >= m) break;
      uint32_t v = bytes[pos / 5];
      for(uint32_t q = (uint32_t)(pos % 5); q; --q) v /= 3;
      if(v % 3 == 2) x |= 1u << b;
    }
    out[w] = x;
  }
}

// Slow path: walk backwards from byte position `end` (exclusive) of the batch collecting
// the symbols emitted before it, newest first, until `need` symbols or a reset is found.
// out[need-1-j] receives the j-th newest symbol, so out[0..need) ends up oldest-first;
// missing leading entries are SYM_BREAK.  `line_nl` = position of the last '\n' before `end`
// if known (>= -1), or -2 when unknown.
template<int CPRE = PRE>               // symbols a Carry holds for this key width
__device__ void backfill_symbols(const uint8_t* in, uint64_t n, const Carry* cin, long long end, long long line_nl,
                                 int need, uint8_t* out, bool keep_cr = false) {
  for(int i = 0; i < need; ++i) out[i] = SYM_BREAK;
  int got = 0;
  long long cur_end = end;           // exclusive end of the line piece under inspection
  long long q = line_nl;
  bool first = true;
  while(got < need) {
    if(!(first && q >= -1)) { q = cur_end - 1; while(q >= 0 && in[q] != '\n') --q; }
    first = false;
    const long long ls = q + 1;      // line start (0 when q == -1: batch start)
    // classify the line
    uint32_t s0 = (q >= 0) ? ST_L : cin->state;
    long long fnc = ls;              // first non-'\r' byte of the line piece (only meaningful when s0 == L)
    uint32_t st = s0;
    if(s0 == ST_L) {
      while(!keep_cr && fnc < cur_end && in[fnc] == '\r') ++fnc;
      st = fnc >= cur_end ? ST_L : (in[fnc] == '>' ? ST_H : ST_S);
    }
    if(st == ST_H) return;           // a header precedes: window reset
    if(st == ST_S) {
      const long long seq_from = (s0 == ST_L) ? fnc : ls;
      for(long long p = cur_end - 1; p >= seq_from && got < need; --p) {
        uint32_t b = in[p];
        uint32_t sy;
        if(b == '\r') { if(!keep_cr && cr_dropped(in, (uint64_t)p, n)) continue; sy = SYM_BREAK; }
        else sy = base_symbol(b);
        if(sy == SYM_BREAK) return;
        out[need - 1 - got] = (uint8_t)sy; ++got;
      }
      if(got >= need) return;
    }
    if(q < 0) {                      // reached the batch start: continue into the previous batch's carry
      for(int j = CPRE - 1; j >= 0 && got < need; --j) {
        uint32_t sy = cin->sym[j];
        if(sy == SYM_BREAK) return;
        out[need - 1 - got] = (uint8_t)sy; ++got;
      }
      return;
    }
    cur_end = q;                     // continue with the previous line (the '\n' itself emits nothing)
  }
}

// FASTQ slow path: a sequence line is never continued from another line, so the symbols before
// `end` are those of the same line (back to its '\n'), then a reset; before the batch start the
// previous batch's carry continues the line.  The caller knows that `end` lies in a sequence line.
// -Q (min_qual != 0): the line is read as K1's per-byte path reads it -- a '\r' resets, and so does a base whose quality
// byte (two lines further down, same column; the line start is looked for at most n_back bytes before the batch) is
// below min_qual as a signed char, or lies at or past n.  Out of line: a cold path that, inlined, made K1 slower.
template<int CPRE = PRE>
__device__ __noinline__ void backfill_fastq(const uint8_t* in, uint64_t n, const Carry* cin, long long end, int need, uint8_t* out,
                               uint32_t min_qual = 0, uint64_t n_back = 0) {
  for(int i = 0; i < need; ++i) out[i] = SYM_BREAK;
  long long qoff = -1;                 // -Q: the quality of the byte at p is in[p + qoff]; -1: none in the text
  if(min_qual && end > 0) {
    long long sl = end - 1; while(sl > -(long long)n_back && in[sl - 1] != '\n') --sl;
    long long e1 = end - 1; while(e1 < (long long)n && in[e1] != '\n') ++e1;
    long long e2 = e1 + 1;  while(e2 < (long long)n && in[e2] != '\n') ++e2;
    if(e2 < (long long)n) qoff = e2 + 1 - sl;
  }
  int got = 0;
  for(long long p = end - 1; got < need; --p) {
    if(p < 0) {
      if((cin->state & 3u) != 1u || (cin->state & 4u)) return;       // the batch did not start inside a sequence line
      for(int j = CPRE - 1; j >= 0 && got < need; --j) {
        const uint32_t sy = cin->sym[j];
        if(sy == SYM_BREAK) return;
        out[need - 1 - got] = (uint8_t)sy; ++got;
      }
      return;
    }
    const uint32_t b = in[p];
    if(b == '\n') return;
    uint32_t sy;
    if(min_qual) sy = (qoff < 0 || p + qoff >= (long long)n || (signed char)in[p + qoff] < (signed char)min_qual) ? (uint32_t)SYM_BREAK : base_symbol(b);
    else if(b == '\r') { if(cr_dropped(in, (uint64_t)p, n)) continue; sy = SYM_BREAK; }
    else sy = base_symbol(b);
    if(sy == SYM_BREAK) return;
    out[need - 1 - got] = (uint8_t)sy; ++got;
  }
}

// ---------------------------------------------------------------------------------------
// K1: the fused counting kernel.  Persistent CTAs; one TMA bulk copy stages a window of
//     NTH*32 bytes (HALO bytes of the previous tile + the tile); the copy of the NEXT window is
//     issued as soon as every thread holds its 32 bytes in registers, so it overlaps the rest.
//
//     MODE 0  insert/increment straight into the table (random HBM access)
//     MODE 1  bucket keys by owning shard for the multi-GPU all-to-all
//     MODE 2  PARTITION: turn every k-mer into a compact record (position-in-region : explicit
//             key bits), stage records per table region in shared memory and append them to
//             per-CTA chunk lists in HBM.  K1b (insert_chunks_kernel) then fills the table one
//             L2-sized region at a time, so the atomics hit L2 instead of random DRAM pages.
// ---------------------------------------------------------------------------------------
constexpr int PMAX        = 2048;          // partitions (table regions) at most
constexpr int CHUNK_BYTES = 8192;          // granule of the record pool
constexpr uint32_t NO_CHUNK = 0xFFFFFFFFu;

// ---- windows of the table and the lazily zeroed table --------------------------------------------
constexpr uint32_t WIN_LG = 14;                    // slots per window (the unit of K2's window form, jf_window.cuh)
constexpr uint32_t WIN_SLOTS = 1u << WIN_LG;
// A table zeroed lazily (jf_engine.cu, table_zero: zero in meaning, garbage in memory until the first drain writes it) keeps one
// state per window.  A kernel that has to insert into it before that drain -- K1 when the spill list is full -- first puts
// every window the probe sequence can reach in memory; the drain then loads those windows instead of overwriting them, and
// table_materialize leaves them alone.
enum : uint32_t { WIN_LAZY = 0, WIN_ZEROING = 1, WIN_IN_MEMORY = 2 };
__device__ __noinline__ void lazy_win_materialize(uint32_t* state, uint32_t* tab, uint64_t local_size, uint64_t first_slot, uint64_t last_slot) {
  const uint64_t w_end = min(last_slot, local_size - 1) >> WIN_LG;          // (the margin past local_size is always in memory)
  for(uint64_t w = first_slot >> WIN_LG; w <= w_end; ++w) {
    volatile uint32_t* s = state + w;
    if(*s == WIN_IN_MEMORY) continue;
    if(atomicCAS(&state[w], WIN_LAZY, WIN_ZEROING) == WIN_LAZY) {
      uint4* p = reinterpret_cast<uint4*>(tab + (w << WIN_LG));
      for(uint32_t i = 0; i < WIN_SLOTS / 4; ++i) p[i] = make_uint4(0, 0, 0, 0);
      __threadfence();
      atomicExch(&state[w], WIN_IN_MEMORY);
    } else {
      while(*s != WIN_IN_MEMORY) __nanosleep(64);   // another thread is zeroing it
    }
  }
  __threadfence();
}

struct PartDev {
  uint32_t  P;              // number of regions (power of two)
  uint32_t  region_bits;    // log2(slots per region)
  uint32_t  rec_bytes;      // 4, 8 or 16
  uint32_t  cap;            // staging capacity per region, records
  uint32_t  flush_min;      // flush a staging buffer holding at least this many records
  uint32_t  chunk_recs;     // records per chunk
  uint32_t  n_chunks;       // chunks in the pool
  uint32_t  stage_bytes;    // shared-memory staging bytes per CTA
  uint32_t  margin;         // a chunk is closed once fewer than `margin` free records remain
  uint32_t  arena_chunks;   // the pool is cut into one arena of this many chunks per CTA of the staging kernels: a CTA's open
                            // chunks then lie within a few MB of each other (its own TLB reach) whatever the other CTAs do
  uint32_t  ring_len;       // records per region ring of the staging kernels (power of two, >= 32): the 128 KB of ring memory
                            // are shared out among the regions, so tables with few regions get long rings
  uint32_t  by_owner;       // sharded counting, send side: regions are those of the GLOBAL table and the arenas belong to the owning
  uint32_t  owner_shift;    // shards (arena = region >> owner_shift), so that a shard's chunks are contiguous for the exchange
  uint32_t* lazy_win;       // the window states of a table zeroed lazily (jf_engine.cu, table_zero), else null: a direct insertion
                            // puts the windows it may reach in memory first (lazy_win_materialize)
  uint8_t*  pool;
  unsigned int* pool_next;  // allocation cursor of every arena
  unsigned int* n_units;    // chunks listed in `order` (written by chunk_scan_kernel)
  uint2*    dir;            // per chunk: { region, records } written when the chunk is closed
  uint32_t* cta_chunk;      // [grid][P] open chunk of each CTA for each region
  uint32_t* cta_fill;       // [grid][P] records already in it
  uint64_t* spill_keys;     // records that found their staging buffer full: inserted directly later
  uint64_t* spill_counts;
  unsigned long long* spill_n;
  uint64_t  spill_cap;
};

// take a fresh chunk from this CTA's arena; NO_CHUNK when the arena is exhausted
__device__ __forceinline__ uint32_t alloc_chunk(const PartDev& pd, uint32_t arena) {
  const uint32_t local = atomicAdd(&pd.pool_next[arena], 1u);
  return local < pd.arena_chunks ? arena * pd.arena_chunks + local : NO_CHUNK;
}
// a fresh chunk from `arena` for a region, with f = 0 records in it; when the arena is exhausted NO_CHUNK, and f = chunk_recs
// sends the region's records to the spill list
__device__ __forceinline__ uint32_t fresh_chunk(const PartDev& pd, uint32_t arena, unsigned long long* stats, uint32_t& f) {
  const uint32_t c = alloc_chunk(pd, arena); f = 0;
  if(c == NO_CHUNK) { atomicAdd(&stats[STAT_POOL_FULL], 1ull); f = pd.chunk_recs; }
  return c;
}
// between two barriers of the staging kernels: close region p's open chunk once fewer than `margin` records are free in it
// and open the next one of this CTA's arena
__device__ __forceinline__ void roll_chunk(const PartDev& pd, uint32_t p, unsigned long long* stats, uint32_t* st_chunk, uint32_t* st_cnt) {
  const uint32_t c = st_cnt[p];
  if(c + pd.margin > pd.chunk_recs) {
    const uint32_t old = st_chunk[p];
    if(old != NO_CHUNK) pd.dir[old] = make_uint2(p, min(c, pd.chunk_recs));
    uint32_t nc = alloc_chunk(pd, blockIdx.x);
    if(nc == NO_CHUNK) { atomicAdd(&stats[STAT_POOL_FULL], 1ull); st_chunk[p] = NO_CHUNK; st_cnt[p] = pd.chunk_recs; }
    else { st_chunk[p] = nc; st_cnt[p] = 0; }
  }
}
__device__ __forceinline__ bool chunk_in_use(const PartDev& pd, uint32_t i) {
  const uint32_t a = i / pd.arena_chunks;
  return i - a * pd.arena_chunks < pd.pool_next[a];
}

// A region record is (position inside the region << hb) | explicit key bits, hb = fbits - rbits; it is stored in
// rec_bytes = 4, 8 or 16 bytes.
__device__ __forceinline__ u128 rec_make(u128 high, uint64_t rel, uint32_t hb) {
  u128 rec;
  if(hb == 0)       { rec.lo = rel; rec.hi = 0; }
  else if(hb < 64)  { rec.lo = high.lo | (rel << hb); rec.hi = high.hi | (rel >> (64 - hb)); }
  else              { rec.lo = high.lo; rec.hi = high.hi | (rel << (hb - 64)); }
  return rec;
}
__device__ __forceinline__ void rec_split(u128 rec, uint32_t hb, u128& high, uint64_t& rel) {
  if(hb == 0)      { rel = rec.lo; high.lo = 0; high.hi = 0; }
  else if(hb < 64) { high.lo = rec.lo & ((1ull << hb) - 1ull); high.hi = 0; rel = (rec.lo >> hb) | (rec.hi << (64 - hb)); }
  else             { high.lo = rec.lo; high.hi = hb == 64 ? 0 : (rec.hi & ((1ull << (hb - 64)) - 1ull)); rel = hb == 64 ? rec.hi : (rec.hi >> (hb - 64)); }
}
__device__ __forceinline__ void store_rec(uint8_t* base, uint32_t rec_bytes, uint32_t idx, u128 r) {
  if(rec_bytes == 4) reinterpret_cast<uint32_t*>(base)[idx] = (uint32_t)r.lo;
  else if(rec_bytes == 8) reinterpret_cast<uint64_t*>(base)[idx] = r.lo;
  else { reinterpret_cast<uint64_t*>(base)[2 * idx] = r.lo; reinterpret_cast<uint64_t*>(base)[2 * idx + 1] = r.hi; }
}
__device__ __forceinline__ u128 load_rec(const uint8_t* base, uint32_t rec_bytes, uint64_t idx) {
  u128 r; r.hi = 0;
  if(rec_bytes == 4) r.lo = reinterpret_cast<const uint32_t*>(base)[idx];
  else if(rec_bytes == 8) r.lo = reinterpret_cast<const uint64_t*>(base)[idx];
  else { r.lo = reinterpret_cast<const uint64_t*>(base)[2 * idx]; r.hi = reinterpret_cast<const uint64_t*>(base)[2 * idx + 1]; }
  return r;
}

// ---------------------------------------------------------------------------------------
// K1b: partitioned insertion.  Chunks are visited region by region (order[] lists the chunk
//      ids sorted by region), every CTA pulling the next chunk from a shared cursor, so that at
//      any moment the whole GPU works on one or two adjacent table regions that sit in L2.
// ---------------------------------------------------------------------------------------
__global__ void close_chunks_kernel(PartDev pd, uint32_t n_cta) {
  for(uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < (uint64_t)n_cta * pd.P; i += (uint64_t)gridDim.x * blockDim.x) {
    const uint32_t c = pd.cta_chunk[i];
    if(c != NO_CHUNK) { pd.dir[c] = make_uint2((uint32_t)(i % pd.P), pd.cta_fill[i]); pd.cta_chunk[i] = NO_CHUNK; pd.cta_fill[i] = 0; }
  }
}
// chunks per region, and records per region unless `recs` is null (only the window form of K2 sizes its groups by records)
__global__ void chunk_hist_kernel(PartDev pd, uint32_t* __restrict__ hist, unsigned long long* __restrict__ recs) {
  for(uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < pd.n_chunks; i += gridDim.x * blockDim.x)
    if(chunk_in_use(pd, i)) {
      const uint2 d = pd.dir[i];
      atomicAdd(&hist[d.x], 1u);
      if(recs) atomicAdd(&recs[d.x], (unsigned long long)d.y);
    }
}
__global__ void __launch_bounds__(1024) chunk_scan_kernel(uint32_t P, const uint32_t* __restrict__ hist, uint32_t* __restrict__ start, uint32_t* __restrict__ cursor,
                                                          unsigned int* __restrict__ n_units) {
  __shared__ uint32_t s[PMAX];
  for(uint32_t p = threadIdx.x; p < P; p += blockDim.x) s[p] = hist[p];
  __syncthreads();
  if(threadIdx.x == 0) { uint32_t run = 0; for(uint32_t p = 0; p < P; ++p) { uint32_t x = s[p]; s[p] = run; run += x; } *n_units = run; }
  __syncthreads();
  for(uint32_t p = threadIdx.x; p < P; p += blockDim.x) { start[p] = s[p]; cursor[p] = s[p]; }
}
__global__ void chunk_scatter_kernel(PartDev pd, uint32_t* __restrict__ cursor, uint32_t* __restrict__ order) {
  for(uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < pd.n_chunks; i += gridDim.x * blockDim.x)
    if(chunk_in_use(pd, i)) order[atomicAdd(&cursor[pd.dir[i].x], 1u)] = i;
}

// A warp works on one 512-byte piece of a chunk at a time (32 lanes x one 128-bit streaming
// load = 128 four-byte records) and takes pieces from ONE shared cursor, so that
//  * the pieces in flight on the whole GPU (~4.7k warps) span only ~300 consecutive chunks of the
//    region-ordered list: one or two table regions, which stay L2 resident;
//  * there is no block-wide barrier: a warp whose keys need long probe sequences delays nobody;
//  * the next piece (cursor, chunk directory, records) is fetched before the current one is
//    inserted, so HBM latency overlaps the probing.
constexpr uint32_t PIECES = CHUNK_BYTES / 512;
constexpr uint32_t PGRAB = 4;      // consecutive pieces a warp takes per visit of the shared cursor

template<int KW, int SB>
__global__ void __launch_bounds__(512, 2) insert_chunks_kernel(TableDev T, PartDev pd, const uint32_t* __restrict__ order,
                                                                unsigned int* __restrict__ piece_cursor, uint32_t from, uint32_t upto,
                                                                const uint64_t* __restrict__ inv_lut_g, uint32_t nbytes) {
  const uint32_t n_units = min(*pd.n_units, upto);
  const uint32_t hb = T.fbits - T.rbits;
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t per16 = 16 / pd.rec_bytes;                         // records per 16 bytes: 4, 2 or 1
  LocalStats ls = { 0, 0, 0, 0, 0 };

  struct Piece { uint4 raw; uint64_t region_base; uint32_t n_rec; uint32_t v0; bool ok; };
  uint32_t g_next = 0, g_left = 0;               // pieces of the current grab still to be fetched
  auto fetch = [&](Piece& pc) {
    if(g_left == 0) {
      uint32_t g0 = 0;
      if(lane == 0) g0 = atomicAdd(piece_cursor, PGRAB);
      g_next = __shfl_sync(0xffffffffu, g0, 0);
      g_left = PGRAB;
    }
    const uint32_t g = g_next++;
    --g_left;
    const uint32_t u = from + g / PIECES;
    pc.ok = u < n_units;
    pc.raw = make_uint4(0, 0, 0, 0); pc.n_rec = 0; pc.v0 = 0; pc.region_base = 0;
    if(!pc.ok) return;
    const uint32_t chunk = order[u];
    const uint2 d = pd.dir[chunk];
    pc.region_base = (uint64_t)d.x << pd.region_bits;
    pc.n_rec = d.y;
    pc.v0 = (g % PIECES) * 32 + lane;
    if(pc.v0 * per16 < d.y) pc.raw = __ldcs(reinterpret_cast<const uint4*>(pd.pool + (size_t)chunk * CHUNK_BYTES) + pc.v0);
  };

  Piece nxt;
  fetch(nxt);
  while(nxt.ok) {
    const Piece cur = nxt;
    fetch(nxt);                                  // in flight while `cur` is inserted
    if(cur.v0 * per16 >= cur.n_rec) continue;
    u128 recs[4]; bool valid[4]; uint64_t base[4]; u128 high[4]; bool ok[4];
    if(pd.rec_bytes == 4) {
      recs[0].lo = cur.raw.x; recs[1].lo = cur.raw.y; recs[2].lo = cur.raw.z; recs[3].lo = cur.raw.w;
      recs[0].hi = recs[1].hi = recs[2].hi = recs[3].hi = 0;
    } else if(pd.rec_bytes == 8) {
      recs[0].lo = (uint64_t)cur.raw.x | ((uint64_t)cur.raw.y << 32); recs[1].lo = (uint64_t)cur.raw.z | ((uint64_t)cur.raw.w << 32);
      recs[0].hi = recs[1].hi = 0; recs[2].lo = recs[2].hi = recs[3].lo = recs[3].hi = 0;
    } else {
      recs[0].lo = (uint64_t)cur.raw.x | ((uint64_t)cur.raw.y << 32); recs[0].hi = (uint64_t)cur.raw.z | ((uint64_t)cur.raw.w << 32);
      recs[1].lo = recs[1].hi = recs[2].lo = recs[2].hi = recs[3].lo = recs[3].hi = 0;
    }
#pragma unroll
    for(int r = 0; r < 4; ++r) {
      valid[r] = (uint32_t)r < per16 && cur.v0 * per16 + r < cur.n_rec;
      uint64_t rel;
      rec_split(recs[r], hb, high[r], rel);
      base[r] = cur.region_base + rel;
    }
    table_add_batch<SB, 4>(T, base, high, valid, ok, ls);
#pragma unroll
    for(int r = 0; r < 4; ++r) {
      if(!valid[r]) continue;
      if(ok[r]) { ls.inserted++; continue; }
      // hash full: rebuild the key for the failure list
      uint64_t key[KW];
      key_from_position<KW>(inv_lut_g, nbytes, T.lsize, high[r], global_pos(T, base[r]), key);
      record_failure<KW>(T, key, 1);
    }
  }
  flush_stats(T.stats, ls.inserted, ls.distinct, ls.reprobes);
}

// ---------------------------------------------------------------------------------------
// K1c: packed keys -> records appended to the per-CTA chunk lists (the receive side of the
//      multi-GPU all-to-all in region-by-region mode: same record pool, same K2 afterwards).
// ---------------------------------------------------------------------------------------
// BF: the --bf-size prefilter of a shard in front of the table, as in insert_keys_bf_kernel; its byte tables follow the
// staging counters in shared memory.  (stage_keys_bf_kernel is instantiated in jf_bloom.cu only.)
template<int KW, bool BF>
__device__ __forceinline__ void stage_keys_body(const TableDev& T, const PartDev& pd, const uint64_t* __restrict__ lut_g, uint32_t nbytes,
                                                const uint64_t* __restrict__ keys, uint64_t n, const BloomDev& B) {
  extern __shared__ __align__(16) uint8_t smem_raw[];
  uint64_t* lut = reinterpret_cast<uint64_t*>(smem_raw);
  uint32_t* st_cnt = reinterpret_cast<uint32_t*>(lut + nbytes * 256);
  uint32_t* st_chunk = st_cnt + PMAX;
  uint64_t* bl1 = reinterpret_cast<uint64_t*>(st_chunk + PMAX);
  uint64_t* bl2 = bl1 + nbytes * 256;
  const int tid = threadIdx.x;
  for(uint32_t i = tid; i < nbytes * 256u; i += blockDim.x) {
    lut[i] = lut_g[i];
    if constexpr(BF) { bl1[i] = B.lut1[i]; bl2[i] = B.lut2[i]; }
  }
  uint32_t* my_chunk = pd.cta_chunk + (size_t)blockIdx.x * pd.P;
  uint32_t* my_fill  = pd.cta_fill + (size_t)blockIdx.x * pd.P;
  for(uint32_t p = tid; p < pd.P; p += blockDim.x) {
    uint32_t c = my_chunk[p], f = my_fill[p];
    if(c == NO_CHUNK) c = fresh_chunk(pd, blockIdx.x, T.stats, f);
    st_chunk[p] = c; st_cnt[p] = f;
  }
  __syncthreads();
  const uint32_t hb = T.fbits - T.rbits;
  // an iteration = 32 keys per thread (the arrival rate the roll-over margin was sized for)
  const uint64_t per_iter = (uint64_t)blockDim.x * 32;
  const uint64_t iters = (n + per_iter * gridDim.x - 1) / (per_iter * gridDim.x);
  for(uint64_t it = 0; it < iters; ++it) {
    const uint64_t base_i = (it * gridDim.x + blockIdx.x) * per_iter;
    for(uint32_t q = 0; q < 32u; ++q) {
      const uint64_t i = base_i + (uint64_t)q * blockDim.x + tid;       // coalesced key loads
      if(i >= n) break;
      uint64_t key[KW];
#pragma unroll
      for(int w = 0; w < KW; ++w) key[w] = keys[i * KW + w];
      if constexpr(BF) {
        if(!bloom_test_and_set(B, gf2_hash<KW>(bl1, key, (int)nbytes), gf2_hash<KW>(bl2, key, (int)nbytes))) continue;
      }
      const uint64_t pos = gf2_hash<KW>(lut, key, (int)nbytes);
      const uint64_t lpos = pos & T.local_mask;
      const uint32_t p = (uint32_t)(lpos >> pd.region_bits);
      const uint64_t rel = lpos & ((1ull << pd.region_bits) - 1ull);
      const u128 rec = rec_make(key_high<KW>(key, T.lsize), rel, hb);
      const uint32_t slot = atomicAdd(&st_cnt[p], 1u);
      if(slot < pd.chunk_recs) store_rec(pd.pool + (size_t)st_chunk[p] * CHUNK_BYTES, pd.rec_bytes, slot, rec);
      else {
        unsigned long long at = atomicAdd(pd.spill_n, 1ull);
        if(at < pd.spill_cap) {
#pragma unroll
          for(int w = 0; w < KW; ++w) pd.spill_keys[at * KW + w] = key[w];
          pd.spill_counts[at] = 1;
        } else atomicAdd(&T.stats[STAT_POOL_FULL], 1ull);
      }
    }
    __syncthreads();
    for(uint32_t p = tid; p < pd.P; p += blockDim.x) roll_chunk(pd, p, T.stats, st_chunk, st_cnt);
    __syncthreads();
  }
  for(uint32_t p = tid; p < pd.P; p += blockDim.x) { my_chunk[p] = st_chunk[p]; my_fill[p] = min(st_cnt[p], pd.chunk_recs); }
}
template<int KW>
__global__ void __launch_bounds__(1024, 1) stage_keys_kernel(TableDev T, PartDev pd, const uint64_t* __restrict__ lut_g, uint32_t nbytes,
                                                              const uint64_t* __restrict__ keys, uint64_t n, uint64_t* __restrict__ spill_keys_unused) {
  stage_keys_body<KW, false>(T, pd, lut_g, nbytes, keys, n, BloomDev());
}
template<int KW>
__global__ void __launch_bounds__(1024, 1) stage_keys_bf_kernel(TableDev T, PartDev pd, const uint64_t* __restrict__ lut_g, uint32_t nbytes,
                                                                 const uint64_t* __restrict__ keys, uint64_t n, BloomDev B) {
  stage_keys_body<KW, true>(T, pd, lut_g, nbytes, keys, n, B);
}

// ---- lean specialisation of K2 for the common geometry: 32-bit slots and 4-byte records ----
// Everything is 32-bit arithmetic except the slot index; rare paths (counter carry, hash full)
// are kept out of line so that the kernel runs with 32 registers, i.e. 2048 threads per SM: the
// kernel is bound by L2 atomic latency, and twice the threads means twice the atomics in flight.
template<int KW>
__device__ __noinline__ void k2_fail(uint32_t shard_index, uint32_t local_lsize, uint32_t lsize, unsigned long long* stats,
                                     uint64_t* fail_keys, uint64_t* fail_counts, uint64_t fail_cap,
                                     uint64_t base, uint32_t high, const uint64_t* inv_lut_g, uint32_t nbytes) {
  // (everything by value, as for spill_record; so the global position is spelled out here rather than taken from global_pos)
  uint64_t key[KW];
  const u128 h = { high, 0 };
  key_from_position<KW>(inv_lut_g, nbytes, lsize, h, ((uint64_t)shard_index << local_lsize) | base, key);
  unsigned long long at = atomicAdd(&stats[STAT_FAILED], 1ull);
  if(at < fail_cap) {
#pragma unroll
    for(int w = 0; w < KW; ++w) fail_keys[at * KW + w] = key[w];
    fail_counts[at] = 1;
  } else atomicAdd(&stats[STAT_FAIL_DROPPED], 1ull);
}
__device__ __noinline__ void k2_carry(unsigned long long* ovf_keys, unsigned long long* ovf_vals, uint64_t ovf_mask, unsigned long long* stats, uint64_t idx) {
  TableDev T; T.ovf_keys = ovf_keys; T.ovf_vals = ovf_vals; T.ovf_mask = ovf_mask; T.stats = stats;
  ovf_add(T, idx, 1);
}

// continue the probe sequence of one key from probe 1 (look-ahead of 4 slots at a time); returns
// false when the reprobe limit is exhausted
// returns 0 = hash full, else 1 + probe index used | (new slot claimed ? 0x10000 : 0) | (counter carry ? 0x20000 : 0)
__device__ __noinline__ uint32_t k2_walk(uint32_t* tab, uint64_t base, uint32_t kf0, uint32_t fb, uint32_t max_reprobe) {
  const uint32_t fmask = (1u << fb) - 1u, one = 1u << fb, cb = 32 - fb;
  for(uint32_t nxt = 1; nxt <= max_reprobe; nxt += 4) {
    uint32_t seen[4];
#pragma unroll
    for(uint32_t j = 0; j < 4; ++j) seen[j] = nxt + j <= max_reprobe ? __ldcg(&tab[base + tri(nxt + j)]) : 0xFFFFFFFFu;
#pragma unroll
    for(uint32_t j = 0; j < 4; ++j) {
      const uint32_t i = nxt + j;
      if(i > max_reprobe) return 0;
      const uint32_t kf = kf0 | (i + 1);
      const uint32_t v = seen[j];
      if(v != 0 && (v & fmask) != kf) continue;
      const uint64_t idx = base + tri(i);
      uint32_t o = v;
      if(v == 0) o = atomicCAS(&tab[idx], 0u, kf | one);
      if(o == 0) return (1 + i) | 0x10000u;
      if((o & fmask) == kf) {
        const uint32_t o2 = atomicAdd(&tab[idx], one);
        return (1 + i) | ((((o2 >> fb) + 1) >> cb) != 0 ? 0x20000u : 0u);
      }
    }
  }
  return 0;
}

// one record of a 32-bit table (slot `base`, explicit key bits `high`) after the CAS of its first probe returned `old`: a
// new key, an increment of the same key (its carry to the side table), or the rest of the probe sequence (k2_walk); a key
// that finds no slot goes to the failure list
template<int KW>
__device__ __forceinline__ void k2_settle(const TableDev& T, uint32_t* tab, uint64_t base, uint32_t high, uint32_t old,
                                          const uint64_t* inv_lut_g, uint32_t nbytes, uint32_t& n_ins, uint32_t& n_new, uint32_t& n_rep) {
  const uint32_t fb = T.fbits, kf0 = high << T.rbits;
  const uint32_t fmask = (1u << fb) - 1u, one = 1u << fb, cb = 32 - fb;
  bool ok = true;
  if(old == 0u) ++n_new;
  else if((old & fmask) == (kf0 | 1u)) {
    const uint32_t o2 = atomicAdd(&tab[base], one);
    if((((o2 >> fb) + 1) >> cb) != 0) k2_carry(T.ovf_keys, T.ovf_vals, T.ovf_mask, T.stats, base);
  } else {
    const uint32_t w = k2_walk(tab, base, kf0, fb, T.max_reprobe);
    ok = w != 0;
    if(ok) {
      const uint32_t i = (w & 0xFFFFu) - 1;
      n_rep += i; if(w & 0x10000u) ++n_new;
      if(w & 0x20000u) k2_carry(T.ovf_keys, T.ovf_vals, T.ovf_mask, T.stats, base + tri(i));
    }
  }
  if(ok) ++n_ins;
  else k2_fail<KW>(T.shard_index, T.local_lsize, T.lsize, T.stats, T.fail_keys, T.fail_counts, T.fail_cap, base, high, inv_lut_g, nbytes);
}

template<int KW>
__global__ void __launch_bounds__(768, 2) insert_chunks32_kernel(TableDev T, PartDev pd, const uint32_t* __restrict__ order,
                                                                   unsigned int* __restrict__ piece_cursor, uint32_t from, uint32_t upto,
                                                                   const uint64_t* __restrict__ inv_lut_g, uint32_t nbytes) {
  const uint32_t n_units = min(*pd.n_units, upto);
  const uint32_t fb = T.fbits, rb = T.rbits, hb = fb - rb;
  const uint32_t one = 1u << fb;
  const uint32_t hmask = hb ? ((1u << hb) - 1u) : 0u;
  const uint32_t lane = threadIdx.x & 31;
  uint32_t* tab = (uint32_t*)T.slots;
  uint32_t n_ins = 0, n_new = 0, n_rep = 0;
  uint32_t g_next = 0, g_left = 0;
  uint4 nraw = make_uint4(0, 0, 0, 0); uint64_t nbase = 0; uint32_t nvalid = 0; bool nok = false;
  auto fetch = [&]() {
    if(g_left == 0) {
      uint32_t g0 = 0;
      if(lane == 0) g0 = atomicAdd(piece_cursor, PGRAB);
      g_next = __shfl_sync(0xffffffffu, g0, 0);
      g_left = PGRAB;
    }
    const uint32_t g = g_next++;
    --g_left;
    const uint32_t u = from + g / PIECES;
    nok = u < n_units; nvalid = 0;
    if(!nok) return;
    const uint32_t chunk = order[u];
    const uint2 d = pd.dir[chunk];
    nbase = (uint64_t)d.x << pd.region_bits;
    const uint32_t v0 = (g % PIECES) * 32 + lane;
    nvalid = v0 * 4 >= d.y ? 0u : min(4u, d.y - v0 * 4);
    if(nvalid) nraw = __ldcs(reinterpret_cast<const uint4*>(pd.pool + (size_t)chunk * CHUNK_BYTES) + v0);
  };
  fetch();
  while(nok) {
    const uint4 raw = nraw; const uint64_t rbase = nbase; const uint32_t nv = nvalid;
    fetch();                                     // next piece in flight while this one is inserted
    if(!nv) continue;
    const uint32_t rec[4] = { raw.x, raw.y, raw.z, raw.w };
    uint32_t old[4];
#pragma unroll
    for(int r = 0; r < 4; ++r)
      old[r] = (uint32_t)r < nv ? atomicCAS(&tab[rbase + (hb < 32 ? rec[r] >> hb : 0u)], 0u, (((rec[r] & hmask) << rb) | 1u) | one) : 1u;
#pragma unroll
    for(int r = 0; r < 4; ++r) {
      if((uint32_t)r >= nv) continue;
      const uint32_t high = rec[r] & hmask;
      k2_settle<KW>(T, tab, rbase + (hb < 32 ? rec[r] >> hb : 0u), high, old[r], inv_lut_g, nbytes, n_ins, n_new, n_rep);
    }
  }
  flush_stats(T.stats, n_ins, n_new, n_rep);
}

// After a regrow in the middle of a drain: the remaining records still describe positions of
// the OLD table (T0).  Rebuild each key with the old inverse matrix, hash it with the new one
// and insert it into the new table.
template<int KW, int SB>
__global__ void __launch_bounds__(512, 1) rehash_chunks_kernel(TableDev T, TableDev T0, PartDev pd, const uint32_t* __restrict__ order,
                                                               unsigned int* __restrict__ unit_cursor, uint32_t from, uint32_t upto,
                                                               const uint64_t* __restrict__ old_inv_g, const uint64_t* __restrict__ new_lut_g,
                                                               uint32_t nbytes) {
  extern __shared__ __align__(16) uint8_t smem_raw[];
  uint64_t* inv = reinterpret_cast<uint64_t*>(smem_raw);
  uint64_t* lut = inv + nbytes * 256;
  for(uint32_t i = threadIdx.x; i < nbytes * 256u; i += blockDim.x) { inv[i] = old_inv_g[i]; lut[i] = new_lut_g[i]; }
  __shared__ uint32_t s_unit;
  __syncthreads();
  const uint32_t n_units = min(*pd.n_units, upto);
  const uint32_t hb = T0.fbits - T0.rbits;
  LocalStats ls = { 0, 0, 0, 0, 0 };
  for(;;) {
    if(threadIdx.x == 0) s_unit = from + atomicAdd(unit_cursor, 1u);
    __syncthreads();
    const uint32_t u = s_unit;
    __syncthreads();
    if(u >= n_units) break;
    const uint32_t chunk = order[u];
    const uint2 d = pd.dir[chunk];
    const uint8_t* src = pd.pool + (size_t)chunk * CHUNK_BYTES;
    const uint64_t region_base = (uint64_t)d.x << pd.region_bits;
    for(uint32_t i = threadIdx.x; i < d.y; i += blockDim.x) {
      u128 high; uint64_t rel;
      rec_split(load_rec(src, pd.rec_bytes, i), hb, high, rel);
      uint64_t key[KW];
      key_from_position<KW>(inv, nbytes, T0.lsize, high, global_pos(T0, region_base + rel), key);
      const uint64_t pos = gf2_hash<KW>(lut, key, (int)nbytes);
      if(table_add<KW, SB>(T, key, pos, 1, ls)) ls.inserted++;
      else record_failure<KW>(T, key, 1);
    }
  }
  flush_stats(T.stats, ls.inserted, ls.distinct, ls.reprobes);
}

// insert the spilled keys (count taken from device memory so that no host round trip is needed)
template<int KW, int SB>
__global__ void __launch_bounds__(256) insert_spill_kernel(TableDev T, const uint64_t* __restrict__ lut_g, uint32_t nbytes, PartDev pd) {
  extern __shared__ __align__(16) uint8_t smem_raw[];
  uint64_t* lut = reinterpret_cast<uint64_t*>(smem_raw);
  for(uint32_t i = threadIdx.x; i < nbytes * 256u; i += blockDim.x) lut[i] = lut_g[i];
  __syncthreads();
  const uint64_t n = min((uint64_t)*pd.spill_n, pd.spill_cap);
  LocalStats ls = { 0, 0, 0, 0, 0 };
  unsigned long long occ = 0;
  for(uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
    uint64_t key[KW];
#pragma unroll
    for(int q = 0; q < KW; ++q) key[q] = pd.spill_keys[i * KW + q];
    const uint64_t pos = gf2_hash<KW>(lut, key, (int)nbytes);
    if(table_add<KW, SB>(T, key, pos, pd.spill_counts[i], ls)) occ += pd.spill_counts[i];
    else record_failure<KW>(T, key, pd.spill_counts[i]);
  }
  flush_stats(T.stats, occ, ls.distinct, ls.reprobes);
}

// ---------------------------------------------------------------------------------------
// K2: packed keys (+ optional counts) -> hash -> insert
// ---------------------------------------------------------------------------------------
template<int KW, int SB>
__global__ void __launch_bounds__(256) insert_keys_kernel(TableDev T, const uint64_t* __restrict__ lut_g, uint32_t nbytes,
                                                          const uint64_t* __restrict__ keys, const uint64_t* __restrict__ counts,
                                                          uint64_t n) {
  extern __shared__ __align__(16) uint8_t smem_raw[];
  uint64_t* lut = reinterpret_cast<uint64_t*>(smem_raw);
  for(uint32_t i = threadIdx.x; i < nbytes * 256u; i += blockDim.x) lut[i] = lut_g[i];
  __syncthreads();
  LocalStats ls = { 0, 0, 0, 0, 0 };
  unsigned long long occ = 0;
  for(uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
    uint64_t key[KW];
#pragma unroll
    for(int q = 0; q < KW; ++q) key[q] = keys[i * KW + q];
    const uint64_t cnt = counts ? counts[i] : 1;
    const uint64_t pos = gf2_hash<KW>(lut, key, (int)nbytes);
    if(table_add<KW, SB>(T, key, pos, cnt, ls)) occ += cnt;
    else { ls.failed++; record_failure<KW>(T, key, cnt); }
  }
  flush_stats(T.stats, occ, ls.distinct, ls.reprobes);
}
// The same with the --bf-size prefilter of a shard in front of the table (sharded counting applies it on the owner, where
// every occurrence of a key arrives; jfgpu_insert_keys): a key reaches the table only when the filter has seen it before.
// The filter's two byte tables follow the table's in shared memory.  (A kernel of its own rather than a template switch of
// the one above, whose code stays as it was; instantiated in jf_bloom.cu only.)
template<int KW, int SB>
__global__ void __launch_bounds__(256) insert_keys_bf_kernel(TableDev T, const uint64_t* __restrict__ lut_g, uint32_t nbytes,
                                                             const uint64_t* __restrict__ keys, uint64_t n, BloomDev B) {
  extern __shared__ __align__(16) uint8_t smem_raw[];
  uint64_t* lut = reinterpret_cast<uint64_t*>(smem_raw);
  uint64_t* bl1 = lut + nbytes * 256;
  uint64_t* bl2 = bl1 + nbytes * 256;
  for(uint32_t i = threadIdx.x; i < nbytes * 256u; i += blockDim.x) { lut[i] = lut_g[i]; bl1[i] = B.lut1[i]; bl2[i] = B.lut2[i]; }
  __syncthreads();
  LocalStats ls = { 0, 0, 0, 0, 0 };
  unsigned long long occ = 0;
  for(uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
    uint64_t key[KW];
#pragma unroll
    for(int q = 0; q < KW; ++q) key[q] = keys[i * KW + q];
    if(!bloom_test_and_set(B, gf2_hash<KW>(bl1, key, (int)nbytes), gf2_hash<KW>(bl2, key, (int)nbytes))) continue;
    const uint64_t pos = gf2_hash<KW>(lut, key, (int)nbytes);
    if(table_add<KW, SB>(T, key, pos, 1, ls)) occ++;
    else { ls.failed++; record_failure<KW>(T, key, 1); }
  }
  flush_stats(T.stats, occ, ls.distinct, ls.reprobes);
}

// ---------------------------------------------------------------------------------------
// K3: collect the records whose ORIGINAL position lies in [seg_lo, seg_hi) (local slot
//     indices).  They live in slots [seg_lo, seg_hi + reprobe margin).  The full key is
//     rebuilt from the stored high bits and the position with the inverse matrix
//     (large_hash_iterator.hpp:164-170; large_hash_array.hpp:851-858).
//     sort key = ((opos - seg_lo) << hb) | high   -- ascending (position, key) order because
//     two keys sharing a position differ in their high bits.
// ---------------------------------------------------------------------------------------
struct CollectArgs {
  TableDev T;
  const uint64_t* inv_lut;     // byte tables of the inverse matrix (low lsize bits of the key)
  uint32_t nbytes;
  uint64_t seg_lo, seg_hi;     // local original positions
  uint64_t scan_hi;            // exclusive end of the slots to scan
  uint64_t lower, upper;       // count filter
  uint32_t hb;                 // number of explicit key bits (2k - lsize, >= 0)
  uint64_t* out_keys;          // KW words per record
  uint64_t* out_counts;
  uint64_t* out_sort_lo;       // low 64 bits of the sort key
  uint64_t* out_sort_hi;       // remaining bits (KW == 2 only; may be NULL)
  unsigned long long* out_n;
  uint64_t out_cap;
};

template<int KW, int SB>
__global__ void __launch_bounds__(256) collect_kernel(const CollectArgs a) {
  extern __shared__ __align__(16) uint8_t smem_raw[];
  uint64_t* lut = reinterpret_cast<uint64_t*>(smem_raw);
  for(uint32_t i = threadIdx.x; i < a.nbytes * 256u; i += blockDim.x) lut[i] = a.inv_lut[i];
  __syncthreads();
  const TableDev& T = a.T;
  const uint32_t lane = threadIdx.x & 31;
  const uint64_t span = a.scan_hi - a.seg_lo;
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  const uint64_t rounds = (span + stride - 1) / stride;
  for(uint64_t r = 0; r < rounds; ++r) {
    const uint64_t i = r * stride + (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const uint64_t idx = a.seg_lo + i;
    bool have = false;
    u128 high; uint32_t rp = 0; uint64_t cnt = 0; uint64_t opos = 0;
    if(i < span && slot_decode<SB>(T, idx, high, rp, cnt)) {
      opos = idx - (rp ? tri(rp) : 0);
      if(opos >= a.seg_lo && opos < a.seg_hi) {
        if(T.stats[STAT_OVERFLOWED]) cnt = slot_full_count<SB>(T, idx, cnt);
        have = cnt >= a.lower && cnt <= a.upper;
      }
    }
    const uint32_t ballot = __ballot_sync(0xffffffffu, have);
    if(ballot) {
      unsigned long long basei = 0;
      if(lane == 0) basei = atomicAdd(a.out_n, (unsigned long long)__popc(ballot));
      basei = __shfl_sync(0xffffffffu, basei, 0);
      if(have) {
        const uint64_t o = basei + __popc(ballot & ((1u << lane) - 1u));
        if constexpr(SB == SB_WIDE) {         // the key is in the slot; the records are only re-inserted (regrow)
          if(o < a.out_cap) {
            const unsigned long long* sl = wide_slot(T, idx);
#pragma unroll
            for(int q = 0; q < 4; ++q) a.out_keys[o * 4 + q] = sl[1 + q];
            a.out_counts[o] = cnt;
            a.out_sort_lo[o] = opos - a.seg_lo;
          }
        } else if(o < a.out_cap) {
          uint64_t key[KW];
          key_from_position<KW>(lut, a.nbytes, T.lsize, high, global_pos(T, opos), key);
#pragma unroll
          for(int q = 0; q < KW; ++q) a.out_keys[o * KW + q] = key[q];
          a.out_counts[o] = cnt;
          const uint64_t rel = opos - a.seg_lo;
          if(KW == 1 || a.out_sort_hi == nullptr) {
            a.out_sort_lo[o] = (a.hb >= 64 ? 0 : (rel << a.hb)) | high.lo;
          } else {
            // 128-bit sort key (rel << hb) | high
            uint64_t lo = high.lo, hi = high.hi;
            if(a.hb < 64) { lo |= rel << a.hb; hi |= a.hb ? (rel >> (64 - a.hb)) : 0; }
            else hi |= rel << (a.hb - 64);
            a.out_sort_lo[o] = lo; a.out_sort_hi[o] = hi;
          }
        }
      }
    }
  }
}

// ---------------------------------------------------------------------------------------
// K5: lookups / histogram straight from the resident table
// ---------------------------------------------------------------------------------------
// array::get_val_for_key (large_hash_array.hpp:384-405): the count of `key` (hashed to `pos`), counter carries included;
// 0 when the key is absent or another shard owns it.  Shared by lookup_kernel and query_lookup_kernel (jf_query.cuh).
template<int KW, int SB>
__device__ __forceinline__ uint64_t table_get(const TableDev& T, const uint64_t (&key)[KW], uint64_t pos, uint32_t shard_bits) {
  const uint32_t owner = shard_bits ? (uint32_t)(pos >> (T.lsize - shard_bits)) : 0u;
  if(owner != T.shard_index) return 0;
  if constexpr(SB == SB_WIDE) {
    uint64_t idx = 0, cnt = 0;
    if(!wide_find(T, pos & T.local_mask, key, idx, cnt)) return 0;
    return T.stats[STAT_OVERFLOWED] ? slot_full_count<SB>(T, idx, cnt) : cnt;
  }
  const u128 want = key_high<KW>(key, T.lsize);
  const uint64_t base = pos & T.local_mask;
  uint64_t idx = base;
  for(uint32_t r = 0; r <= T.max_reprobe; ++r) {
    u128 high; uint32_t rp; uint64_t cnt;
    if(!slot_decode<SB>(T, idx, high, rp, cnt)) break;          // empty slot ends the probe sequence
    if(rp == r && high.lo == want.lo && high.hi == want.hi) {
      if(T.stats[STAT_OVERFLOWED]) cnt = slot_full_count<SB>(T, idx, cnt);
      return cnt;
    }
    idx = base + tri(r + 1);
  }
  return 0;
}

template<int KW, int SB>
__global__ void __launch_bounds__(256) lookup_kernel(TableDev T, const uint64_t* __restrict__ lut_g, uint32_t nbytes,
                                                     const uint64_t* __restrict__ keys, uint64_t n, uint64_t* __restrict__ vals,
                                                     uint32_t shard_bits) {
  extern __shared__ __align__(16) uint8_t smem_raw[];
  uint64_t* lut = reinterpret_cast<uint64_t*>(smem_raw);
  for(uint32_t i = threadIdx.x; i < nbytes * 256u; i += blockDim.x) lut[i] = lut_g[i];
  __syncthreads();
  for(uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
    uint64_t key[KW];
#pragma unroll
    for(int q = 0; q < KW; ++q) key[q] = keys[i * KW + q];
    const uint64_t pos = gf2_hash<KW>(lut, key, (int)nbytes);
    vals[i] = table_get<KW, SB>(T, key, pos, shard_bits);
  }
}

template<int SB>
__global__ void __launch_bounds__(256) histogram_kernel(TableDev T, uint64_t n_slots, unsigned long long* __restrict__ hist, uint32_t n_bins) {
  for(uint64_t idx = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < n_slots; idx += (uint64_t)gridDim.x * blockDim.x) {
    u128 high; uint32_t rp; uint64_t cnt;
    if(slot_decode<SB>(T, idx, high, rp, cnt)) {
      if(T.stats[STAT_OVERFLOWED]) cnt = slot_full_count<SB>(T, idx, cnt);
      atomicAdd(&hist[cnt < n_bins ? cnt : n_bins - 1], 1ull);
    }
  }
}

template<int SB>
__global__ void __launch_bounds__(256) max_count_kernel(TableDev T, uint64_t n_slots) {
  unsigned long long m = 0;
  for(uint64_t idx = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < n_slots; idx += (uint64_t)gridDim.x * blockDim.x) {
    u128 high; uint32_t rp; uint64_t cnt;
    if(slot_decode<SB>(T, idx, high, rp, cnt)) {
      if(T.stats[STAT_OVERFLOWED]) cnt = slot_full_count<SB>(T, idx, cnt);
      m = max(m, (unsigned long long)cnt);
    }
  }
#pragma unroll
  for(int o = 16; o; o >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, o));
  if((threadIdx.x & 31) == 0 && m) atomicMax(&T.stats[STAT_MAXCOUNT], m);
}

// ---------------------------------------------------------------------------------------
// synthetic FASTA of the shape jellyfish/generate_sequence.cc:119-149 writes:
// ">read1\n" then 70 bases per line.  Base i is drawn from a counter-based generator
// (splitmix64 of seed + i/32 gives 32 bases), so any byte range can be generated independently.
// ---------------------------------------------------------------------------------------
__host__ __device__ __forceinline__ uint64_t splitmix64(uint64_t x) {
  x += 0x9E3779B97F4A7C15ull;
  x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
  x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
  return x ^ (x >> 31);
}
constexpr int SYNTH_HDR = 7;     // strlen(">read1\n")
constexpr int SYNTH_LINE = 70;

__global__ void __launch_bounds__(256) synth_fasta_kernel(uint8_t* __restrict__ out, uint64_t n_bytes, uint64_t n_bases, uint64_t seed) {
  const char hdr[SYNTH_HDR + 1] = ">read1\n";
  for(uint64_t p = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; p < n_bytes; p += (uint64_t)gridDim.x * blockDim.x) {
    uint8_t c;
    if(p < SYNTH_HDR) c = (uint8_t)hdr[p];
    else {
      const uint64_t q = p - SYNTH_HDR;
      const uint64_t line = q / (SYNTH_LINE + 1), col = q % (SYNTH_LINE + 1);
      if(col == SYNTH_LINE) c = '\n';
      else {
        const uint64_t i = line * SYNTH_LINE + col;
        if(i >= n_bases) c = '\n';
        else {
          const uint64_t r = splitmix64(seed + (i >> 5));
          c = (uint8_t)"ACGT"[(r >> (2 * (i & 31))) & 3];
        }
      }
    }
    out[p] = c;
  }
}

}  // namespace jfk
#endif
