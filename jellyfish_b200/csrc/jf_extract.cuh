// jf_extract.cuh -- K1, the fused extraction kernel (second generation).
//
// Same contract as the first-generation count_kernel (text semantics of
// mer_overlap_sequence_parser.hpp:161-185,260-287, canonical k-mers of mer_dna.hpp:322-370, GF(2) hash of
// rectangular_binary_matrix.hpp:223-261) with the per-byte work replaced by word-parallel work:
//
//   * classification: 4 bytes at a time.  The 2-bit code of a byte is ((b>>1)^(b>>2))&3; whether the
//     byte really is one of ACGTacgt is checked by looking the expected letter up with PRMT (a 4-entry
//     byte table indexed by the code) and comparing all four bytes at once.  Only the bytes that are NOT
//     bases (newlines, header characters, N...) are inspected individually;
//   * the parser state machine works on 32-bit masks (newlines, '>' at a line start, header spans);
//     the per-byte loops survive only for pieces containing '\r' (look-ahead semantics) and for FASTQ;
//   * symbols are compacted into a 2-bit packed stream (+ a 1-bit "window reset" stream) in shared
//     memory with 32-bit atomicOr, three per thread, instead of one byte store per symbol;
//   * a thread then owns one aligned 32-symbol word of the stream: the forward k-mer ending at each of
//     its symbols is a funnel shift of the pair-reversed words, the reverse complement is the complement
//     of a funnel shift of the words as they are -- no rolling, no per-symbol branches; the k-mers that
//     contain a reset are masked out with a dilated copy of the reset stream.
#ifndef JF_EXTRACT_CUH
#define JF_EXTRACT_CUH
#include "jf_kernels.cuh"

// JF_K1_PROF=1 (only in the build scripts/k1_phases.py makes for itself): the FAST kernels stamp clock64() around each
// block barrier and add, per warp, the cycles spent working in each segment and waiting at the barrier that ends it to
// k1_prof_acc.  The product build leaves it at 0, and every kernel there compiles as if the stamps did not exist.
#ifndef JF_K1_PROF
#define JF_K1_PROF 0
#endif

namespace jfk {

// segments of a window, each ended by a block barrier: TMA wait, B, C (scan), C (stream OR), D, E appends (4 per window),
// ring passes (4 per window), E end, window end.  k1_prof_acc: work and wait cycles of every segment summed over warps, then
// the hashing part of the E appends (per warp, no barrier), the warp-cycles of the window loop, windows, CTAs
enum { K1P_TMA, K1P_B, K1P_C, K1P_OR, K1P_D, K1P_APPEND, K1P_PASS, K1P_EEND, K1P_WEND, K1P_SEGS };
constexpr int K1P_WORDS = 2 * K1P_SEGS + 4;
#if JF_K1_PROF
static __device__ unsigned long long k1_prof_acc[K1P_WORDS];
#endif

// PREN = symbol positions kept in front of the window: PRE, or PRE_WIDE for four-word keys
template<int NTH, int PREN = PRE>
struct __align__(16) ExtractSmemT {
  uint8_t  win[NTH * 32];            // TMA destination
  uint32_t rev[2 * (NTH + PREN / 32 + 2)];   // 2-bit symbol stream, little endian: symbol s at bits 2(s&15) of rev[s>>4]
  uint32_t brk[NTH + PREN / 32 + 2];         // reset stream: bit (s&31) of brk[s>>5]
  uint8_t  pre[PREN];                // byte symbols of the PREN stream positions in front of the window
  uint64_t bar;
  uint32_t warp_fn[NTH / 32];
  uint32_t warp_cnt[NTH / 32];
  uint32_t idx0, nsym, halo_break, total_state;
  unsigned long long part[NTH / 32][4];
};

__device__ __forceinline__ uint32_t low_mask32(uint32_t n) { return n >= 32 ? 0xFFFFFFFFu : ((1u << n) - 1u); }
__device__ __forceinline__ uint64_t low_mask64(uint32_t n) { return n >= 64 ? ~0ull : ((1ull << n) - 1ull); }

// reverse the order of the 32 two-bit symbols of a 64-bit word
__device__ __forceinline__ uint64_t pair_reverse64(uint64_t x) {
  uint32_t lo = __brev((uint32_t)(x >> 32)), hi = __brev((uint32_t)x);
  lo = ((lo >> 1) & 0x55555555u) | ((lo & 0x55555555u) << 1);
  hi = ((hi >> 1) & 0x55555555u) | ((hi & 0x55555555u) << 1);
  return ((uint64_t)hi << 32) | lo;
}

// classify the four bytes of w: bit i of the result = byte i is one of ACGTacgt;
// codes = the four 2-bit codes packed into 8 bits (garbage for bytes that are not bases)
__device__ __forceinline__ uint32_t classify4(uint32_t w, uint32_t& codes) {
  const uint32_t x = (w >> 1) & 0x03030303u;
  const uint32_t c = x ^ ((x >> 1) & 0x01010101u);              // A,a->0 C,c->1 G,g->2 T,t->3 (mer_dna.hpp:38-55)
  const uint32_t t = c | (c >> 4);
  const uint32_t sel = __byte_perm(t, 0u, 0x4420u);             // nibble i = code of byte i
  const uint32_t expect = __byte_perm(0x54474341u, 0u, sel);    // the upper-case letter with that code
  const uint32_t d = (w & 0xDFDFDFDFu) ^ expect;                // zero byte <=> the byte is that letter (either case)
  const uint32_t z = ~(((d & 0x7F7F7F7Fu) + 0x7F7F7F7Fu) | d | 0x7F7F7F7Fu);   // 0x80 in every zero byte (exact)
  codes = (c * 0x01041040u) >> 24;
  return ((z >> 7) * 0x10204080u) >> 28;
}

// delete the symbols whose bit is set in `del` from a 2-bit stream `c` and a 1-bit stream `b` (runs, highest first)
__device__ __forceinline__ void squeeze(uint64_t& c, uint32_t& b, uint32_t del) {
  while(del) {
    const uint32_t top = 31 - __clz(del);
    const uint32_t len = __clz(~(del << (31 - top)));            // length of the run of ones ending at `top`
    const uint32_t a = top + 1 - len;
    const uint64_t lm = low_mask64(2 * a);
    c = (c & lm) | (2 * (top + 1) >= 64 ? 0ull : ((c >> (2 * len)) & ~lm));
    const uint32_t l32 = low_mask32(a);
    b = (b & l32) | (top + 1 >= 32 ? 0u : ((b >> len) & ~l32));
    del &= l32;
  }
}

// A region's open chunk filled up inside one window (skewed input): the key goes to the spill list, which K2 inserts
// directly after the regions; out of line, it is a cold path.
template<int KW, int SB>
__device__ __noinline__ void spill_record(const TableDev T, uint64_t* spill_keys, uint64_t* spill_counts, unsigned long long* spill_n, uint64_t spill_cap,
                                          uint64_t k0, uint64_t k1, uint64_t pos, uint32_t* lazy_win) {
  // (everything by value: taking the address of the kernel's parameter structures would move them to local memory)
  uint64_t key[KW];
  key[0] = k0; if(KW == 2) key[KW - 1] = k1;
  unsigned long long at = atomicAdd(spill_n, 1ull);
  if(at < spill_cap) {
#pragma unroll
    for(int q = 0; q < KW; ++q) spill_keys[at * KW + q] = key[q];
    spill_counts[at] = 1;
    return;
  }
  // the list is full as well: insert right here (statistics straight to the global counters: the caller's stay in registers)
  if(SB == 32 && lazy_win) {                       // (only tables of 32-bit slots are zeroed lazily)
    const uint64_t p = pos & T.local_mask;
    lazy_win_materialize(lazy_win, (uint32_t*)T.slots, T.local_mask + 1, p, p + tri(T.max_reprobe));
  }
  LocalStats l = { 0, 0, 0, 0, 0 };
  if(table_add<KW, SB>(T, key, pos, 1, l)) {
    atomicAdd(&T.stats[STAT_INSERTED], 1ull);
    if(l.distinct) atomicAdd(&T.stats[STAT_DISTINCT], (unsigned long long)l.distinct);
    if(l.reprobes) atomicAdd(&T.stats[STAT_REPROBES], (unsigned long long)l.reprobes);
  } else record_failure<KW>(T, key, 1);
}

// FAST = the common geometry of the region-by-region path, everything in 32-bit arithmetic: one key word, the
// 11-bit-table hash with at most six parity rows (tables of up to 2^38 slots), 4-byte records, at most RING_P regions
// (the regions of this GPU's table, or -- sharded counting -- of the GLOBAL table, chunks then grouped by owning shard).  Its records do not go to the chunks one 4-byte store at a time (the GPU retires ~98 G scattered stores
// per second whatever their width, scripts/micro/scatter_store.cu -- that alone would cap K1 at 98 G k-mers/s): every region
// has a ring of RING records in shared memory, and after every 8 k-mers per thread (SG on the sharded send side) a pass over
// the regions writes the complete groups of 8 records with two 16-byte stores (one 32-byte sector).
constexpr uint32_t RING = 32;                     // records per region ring with RING_P regions (PartDev::ring_len in general)
constexpr uint32_t RING_P = 1024;                 // regions at most on the FAST path (shared memory: RING_P * RING * 4 bytes)
// shared memory of the FAST tail behind the hash table: per region a counter, an open chunk id and a ring; then the arena cursor
constexpr size_t FAST_SMEM = (size_t)RING_P * 8 + (size_t)RING_P * RING * 4 + 16;
// NPR (FAST only): parity rows evaluated per k-mer -- 2 covers tables of up to 2^34 slots (unused rows are zero), 6 the
// sharded tables of up to 2^38.
template<int KW, int SB, int MODE, int NTH, bool FAST, int NPR = 2>
__global__ void __launch_bounds__(NTH, (NTH == 512 ? 2 : 1)) extract_kernel(const CountArgs a, const PartDev pd) {
  constexpr int WINB = NTH * 32;
  constexpr int TILEB = WINB - HALO;
  constexpr int NW = NTH / 32;
  constexpr int PREK = KW == 4 ? PRE_WIDE : PRE;  // symbol positions in front of the window (>= k - 1)
  constexpr int PW = PREK / 32;                  // 64-bit stream words in front of the window (PREK symbols)
  constexpr int SG = 4;                          // k-mers whose shared-memory round trips are kept in flight together (FAST tail)
  extern __shared__ __align__(16) uint8_t smem_raw[];
  ExtractSmemT<NTH, PREK>& sm = *reinterpret_cast<ExtractSmemT<NTH, PREK>*>(smem_raw);
  uint64_t* lut = reinterpret_cast<uint64_t*>(smem_raw + ((sizeof(ExtractSmemT<NTH, PREK>) + 15) & ~(size_t)15));
  // per region: records in the open chunk (FAST: low 16 bits = records handed out, high 16 bits = records already written to
  // the chunk) and the open chunk's id; FAST: the rings behind them
  uint32_t* st_cnt = reinterpret_cast<uint32_t*>(reinterpret_cast<uint8_t*>(lut) + a.lut_bytes);
  uint32_t* st_chunk = st_cnt + (FAST ? RING_P : PMAX);
  uint32_t* ring = st_chunk + RING_P;            // (FAST only)
  // FAST, single-GPU counting: the allocation cursor of this CTA's arena, kept here for the launch.  Arena blockIdx.x is this
  // CTA's alone, and the K1 launches of one engine run one after the other on one stream (the open chunks in cta_chunk rely
  // on that too), so closing a chunk costs a shared-memory atomic instead of a round trip to L2 while 1023 threads wait at
  // the next barrier.  The sharded send side shares each owner's arena among all CTAs and keeps the global cursor.
  unsigned int* arena_next = ring + RING_P * RING;
  const bool own_arena = FAST && !pd.by_owner;
  // byte tables of the two Bloom hash matrices, behind everything else
  uint64_t* bl1 = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(lut) + a.lut_bytes +
                                              (MODE == 2 ? (FAST ? FAST_SMEM : (size_t)PMAX * 8) : 0));
  uint64_t* bl2 = bl1 + a.nbytes * 256;
  const uint32_t* lut32 = reinterpret_cast<const uint32_t*>(lut);
  const uint64_t* rev64 = reinterpret_cast<const uint64_t*>(sm.rev);

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const uint32_t k = a.k;
  const uint64_t n = a.n;
#if JF_K1_PROF
  constexpr bool PROF = FAST;
  __shared__ unsigned long long prof_w[NW][2 * K1P_SEGS + 2];   // per warp: work and wait cycles per segment, hashing, loop
  long long prof_t = 0;                                          // when this warp left the last barrier
  if(PROF && tid < NW * (2 * K1P_SEGS + 2)) (&prof_w[0][0])[tid] = 0;
#endif
  // a block barrier that ends segment s of a window (JF_K1_PROF: timed)
  auto bsync = [&](const int s) {
#if JF_K1_PROF
    if constexpr(PROF) {
      const long long t0 = clock64();
      __syncthreads();
      const long long t1 = clock64();
      if(lane == 0) { prof_w[warp][2 * s] += t0 - prof_t; prof_w[warp][2 * s + 1] += t1 - t0; }
      prof_t = t1;
      return;
    }
#endif
    (void)s;
    __syncthreads();
  };

  for(uint32_t i = tid; i < a.lut_bytes / 8; i += NTH) lut[i] = a.lut[i];
  if(a.bloom.mode) for(uint32_t i = tid; i < a.nbytes * 256; i += NTH) { bl1[i] = a.bloom.lut1[i]; bl2[i] = a.bloom.lut2[i]; }
  uint32_t* my_chunk = MODE == 2 ? pd.cta_chunk + (size_t)blockIdx.x * pd.P : nullptr;
  uint32_t* my_fill  = MODE == 2 ? pd.cta_fill + (size_t)blockIdx.x * pd.P : nullptr;
  // FAST: a fresh chunk for region p; NO_CHUNK when the arena is exhausted
  auto take_chunk = [&](const uint32_t p) -> uint32_t {
    if(!own_arena) return alloc_chunk(pd, pd.by_owner ? (p >> pd.owner_shift) : blockIdx.x);
    const uint32_t local = atomicAdd(arena_next, 1u);
    return local < pd.arena_chunks ? blockIdx.x * pd.arena_chunks + local : NO_CHUNK;
  };
  if(MODE == 2) {
    if(own_arena) {
      if(tid == 0) *arena_next = pd.pool_next[blockIdx.x];
      __syncthreads();
    }
    for(uint32_t p = tid; p < pd.P; p += NTH) {
      uint32_t c = my_chunk[p], f = my_fill[p];
      if(c == NO_CHUNK) {
        if constexpr(FAST) {
          c = take_chunk(p); f = 0;
          if(c == NO_CHUNK) { atomicAdd(&a.T.stats[STAT_POOL_FULL], 1ull); f = pd.chunk_recs; }
        } else c = fresh_chunk(pd, pd.by_owner ? (p >> pd.owner_shift) : blockIdx.x, a.T.stats, f);
      }
      st_chunk[p] = c; st_cnt[p] = FAST ? (f | (f << 16)) : f;
    }
  }
  // FAST: one pass over the regions -- write the complete groups of 8 records of every ring to its chunk, close chunks that are
  // nearly full.  Between two barriers; `finish` also writes the incomplete group (end of the launch).
  // Two threads per region: each group goes out as the two 16-byte halves of one 32-byte sector, written by neighbouring
  // lanes in one store instruction, so it costs one store request instead of two; that took a third off the passes' time
  // (DESIGN.md section 6, "K1 phase by phase").
  const uint32_t rlen = pd.ring_len;
  // the word of slot s of region p's ring.  Every ring starts at bank 0 and a pass reads the rings of consecutive regions
  // in 16-byte pieces at fill levels that are multiples of 8, which would touch only every other group of 4 banks: ring p is
  // rotated by 4 (p & 7) words so that they touch all of them
  auto ring_word = [&](const uint32_t p, const uint32_t s) -> uint32_t { return p * rlen + ((s + 4u * (p & 7u)) & (rlen - 1)); };
  auto flush_rings = [&](const bool finish) {
    const uint32_t half = tid & 1u;                // which 16 bytes of a group this thread writes
    // (every thread runs the same iterations, so the whole warp can meet at __syncwarp)
    for(uint32_t base = 0; base < pd.P; base += NTH / 2) {
      const uint32_t p = base + (tid >> 1);
      const bool live = p < pd.P;
      const uint32_t v = live ? st_cnt[p] : 0u;
      uint32_t cnt = v & 0xFFFFu, fl = v >> 16;
      const uint32_t lim = min(fl + rlen, pd.chunk_recs);
      if(cnt > lim) cnt = lim;                    // the slots beyond went to the spill list: hand them out again
      const uint32_t c = live ? st_chunk[p] : NO_CHUNK;
      uint32_t* dst = reinterpret_cast<uint32_t*>(pd.pool + (size_t)c * CHUNK_BYTES);
      if(c != NO_CHUNK) {
        // (only after a launch that ended inside a group; both threads store the same words)
        while((fl & 7u) && fl < cnt) { dst[fl] = ring[ring_word(p, fl)]; ++fl; }
        while(cnt - fl >= 8u) {
          const uint32_t s = fl + 4u * half;
          *reinterpret_cast<uint4*>(dst + s) = *reinterpret_cast<const uint4*>(ring + ring_word(p, s));
          fl += 8;
        }
      }
      // the rest of the region's pass is the first thread's: its writes of st_cnt[p] and st_chunk[p] wait until the second
      // thread has read them
      __syncwarp();
      if(half || c == NO_CHUNK) continue;
      const bool close = cnt + min(rlen, pd.margin) > pd.chunk_recs;
      if(close || finish) for(; fl < cnt; ++fl) dst[fl] = ring[ring_word(p, fl)];
      if(close) {
        pd.dir[c] = make_uint2(p, cnt);
        const uint32_t nc = take_chunk(p);
        st_chunk[p] = nc;
        if(nc == NO_CHUNK) { atomicAdd(&a.T.stats[STAT_POOL_FULL], 1ull); cnt = fl = pd.chunk_recs; }
        else cnt = fl = 0;
      }
      st_cnt[p] = cnt | (fl << 16);
    }
  };
  for(uint32_t i = tid; i < 2 * (NTH + PW + 2); i += NTH) sm.rev[i] = 0;
  for(uint32_t i = tid; i < NTH + PW + 2; i += NTH) sm.brk[i] = 0;
  if(tid == 0) mbar_init(&sm.bar, 1);
  __syncthreads();
#if JF_K1_PROF
  const long long prof_start = clock64();
  prof_t = prof_start;
#endif

  auto issue = [&](uint64_t t) {       // TMA copy of window t (thread 0 only)
    long long h = (long long)(t * (uint64_t)TILEB) - HALO;
    long long from = h < 0 ? 0 : h;
    uint64_t avail = n - (uint64_t)from;
    uint64_t want = (uint64_t)((h + WINB) - from);
    uint32_t bytes = (uint32_t)((avail < want ? avail : want) & ~(uint64_t)15);
    if(bytes) { mbar_expect_tx(&sm.bar, bytes); tma_load_1d(&sm.win[from - h], a.in + from, bytes, &sm.bar); }
    else mbar_arrive(&sm.bar);
  };

  LocalStats ls = { 0, 0, 0, 0, 0 };
  uint32_t phase = 0;
  uint64_t t = blockIdx.x;
  if(t < a.n_tiles && tid == 0) issue(t);

  // constants of the 32-bit tail (FAST)
  const uint32_t f_rgb = pd.region_bits, f_hb = a.T.fbits - a.T.rbits, f_lsz = a.T.lsize;
  const uint32_t f_relmask = f_rgb >= 32 ? 0xFFFFFFFFu : ((1u << f_rgb) - 1u);
  // constants of the k-mer extraction
  const uint32_t kbits = 2 * k;
  const uint64_t kmask_lo = kbits >= 64 ? ~0ull : ((1ull << kbits) - 1ull);
  const uint64_t kmask_hi = KW == 1 ? 0ull : (kbits >= 128 ? ~0ull : ((1ull << (kbits - 64)) - 1ull));

  for(; t < a.n_tiles; t += gridDim.x) {
    const long long h = (long long)(t * (uint64_t)TILEB) - HALO;      // global position of window byte 0
    const long long wend_ll = (long long)n < h + WINB ? (long long)n : h + WINB;
    {   // tail bytes that the 16-byte granular TMA copy left out
      long long from = h < 0 ? 0 : h;
      long long copied = ((wend_ll - from) & ~15ll);
      long long g = from + copied + tid;
      if(tid < 16 && g < wend_ll) sm.win[g - h] = a.in[g];
    }
    mbar_wait(&sm.bar, phase);
    phase ^= 1;
    bsync(K1P_TMA);

    // ---- phase B: 32 bytes per thread, word-parallel classification ----
    uint32_t w[8];
    {
      const uint4* p4 = reinterpret_cast<const uint4*>(sm.win + tid * 32);
      uint4 x0 = p4[0], x1 = p4[1];
      w[0] = x0.x; w[1] = x0.y; w[2] = x0.z; w[3] = x0.w; w[4] = x1.x; w[5] = x1.y; w[6] = x1.z; w[7] = x1.w;
    }
    const long long g0 = h + (long long)tid * 32;       // global position of this thread's first byte
    int vlo = g0 < 0 ? (int)(-g0 < 32 ? -g0 : 32) : 0;
    int vhi = (wend_ll - g0) < 0 ? 0 : ((wend_ll - g0) > 32 ? 32 : (int)(wend_ll - g0));
    if(vhi < vlo) vhi = vlo;
    const uint32_t live = low_mask32((uint32_t)vhi) & ~low_mask32((uint32_t)vlo);

    uint32_t V = 0; uint64_t C = 0;
#pragma unroll
    for(int j = 0; j < 8; ++j) {
      uint32_t codes;
      const uint32_t vm = classify4(w[j], codes);
      V |= vm << (4 * j);
      C |= (uint64_t)codes << (8 * j);
    }
    // the bytes that are not bases, one by one: newline, '>' and '\r' masks
    uint32_t N = 0, Gm = 0, Rm = 0;
    for(uint32_t r = live & ~V; r; r &= r - 1) {
      const uint32_t p = __ffs(r) - 1;
      const uint32_t b = sm.win[tid * 32 + p];
      N |= (uint32_t)(b == '\n') << p; Gm |= (uint32_t)(b == '>') << p; Rm |= (uint32_t)(b == '\r') << p;
    }
    if(a.min_qual) Rm = 0;                               // -Q: std::getline keeps '\r' in the sequence, where it resets the window
    const bool slow = a.format == 1 || Rm != 0;          // per-byte path: FASTQ line types, '\r' look-ahead

    uint32_t prevb = 'x';
    if(a.format == 1 && vhi > vlo) {
      const long long gp = g0 + vlo - 1;
      if(gp < 0) prevb = (a.carry_in->state & 4u) ? '\n' : 'x';
      else if(tid * 32 + vlo - 1 >= 0) prevb = sm.win[tid * 32 + vlo - 1];
      else prevb = a.in[gp];
    }
    uint32_t f;
    if(a.format == 1) f = fn_rot(__popc(N));
    else if(live == 0) f = FN_ID;
    else if(!slow) {
      if(N) {
        const uint32_t last_nl = 31 - __clz(N);
        const uint32_t after = last_nl >= 31 ? 0u : (live & ~((2u << last_nl) - 1u));
        const uint32_t st = !after ? (uint32_t)ST_L : (((Gm >> (__ffs(after) - 1)) & 1u) ? (uint32_t)ST_H : (uint32_t)ST_S);
        f = fn_const(st);
      } else {
        const uint32_t fl = ((Gm >> (__ffs(live) - 1)) & 1u) ? (uint32_t)ST_H : (uint32_t)ST_S;
        f = (uint32_t)ST_H | ((uint32_t)ST_S << 2) | (fl << 4) | (3u << 6);
      }
    } else {
      uint32_t st = ST_L; bool seen_nl = false;
#pragma unroll 1
      for(int i = vlo; i < vhi; ++i) {
        const uint32_t b = sm.win[tid * 32 + i];
        if(b == '\n') { st = ST_L; seen_nl = true; }
        else if(st == ST_L && b != '\r') st = (b == '>') ? ST_H : ST_S;
      }
      f = seen_nl ? fn_const(st) : ((uint32_t)ST_H | ((uint32_t)ST_S << 2) | (st << 4) | (3u << 6));
    }
    uint32_t inc = f;
#pragma unroll
    for(int o = 1; o < 32; o <<= 1) {
      uint32_t up = __shfl_up_sync(0xffffffffu, inc, o);
      if(lane >= o) inc = fn_compose(up, inc);
    }
    if(lane == 31) sm.warp_fn[warp] = inc;
    bsync(K1P_B);
    uint32_t entry = (t == 0) ? (a.format == 1 ? (a.carry_in->state & 3u) : a.carry_in->state) : (uint32_t)a.tile_state[t];
    uint32_t wpre;
    {   // composition of the functions of the warps in front of this one: every warp scans the NW partials itself
      uint32_t g = lane < NW ? sm.warp_fn[lane] : FN_ID;
#pragma unroll
      for(int o = 1; o < NW; o <<= 1) {
        uint32_t up = __shfl_up_sync(0xffffffffu, g, o);
        if(lane >= o) g = fn_compose(up, g);
      }
      wpre = __shfl_sync(0xffffffffu, g, warp ? warp - 1 : 0);
      if(warp == 0) wpre = FN_ID;
    }
    uint32_t excl = __shfl_up_sync(0xffffffffu, inc, 1);
    if(lane == 0) excl = FN_ID;
    const uint32_t st_in = fn_apply(fn_compose(wpre, excl), entry);
    if(tid == NTH - 1) sm.total_state = fn_apply(fn_compose(wpre, inc), entry);

    // ---- phase C: the symbols this thread emits: 2-bit codes `sy`, reset bits `bk`, `cnt` of them ----
    uint64_t sy = 0; uint32_t bk = 0, cnt = 0;
    if(!slow) {
      const uint32_t ls_bits = ((N << 1) | (st_in == (uint32_t)ST_L ? (live & (0u - live)) : 0u)) & live;   // bytes at a line start
      const uint32_t GS = Gm & ls_bits;                                          // header starts
      uint32_t Hm = 0;
      if(st_in == (uint32_t)ST_H) Hm = live & low_mask32(N ? (uint32_t)(__ffs(N) - 1) : 32u);
      for(uint32_t g = GS; g; g &= g - 1) {
        const uint32_t s = __ffs(g) - 1;
        const uint32_t above = N & ~low_mask32(s);
        Hm |= low_mask32(above ? (uint32_t)(__ffs(above) - 1) : 32u) & ~low_mask32(s);
      }
      const uint32_t E = live & ~N & ~(Hm & ~GS);
      sy = C; bk = E & ~V; cnt = __popc(E);
      squeeze(sy, bk, ~E);
    } else if(a.format == 1) {
      // FASTQ, 4-line records (mer_overlap_sequence_parser.hpp:187-217): only sequence lines emit symbols; the
      // start of a header line emits the window reset; '@' / '+' at the line starts are verified
      uint32_t ty = st_in; bool at_start = prevb == '\n';
      long long qoff = 0; bool have_q = false;      // -Q: quality of the sequence byte at global position g is in[g + qoff]
#pragma unroll 1
      for(int i = vlo; i < vhi; ++i) {
        {
          const uint32_t b = sm.win[tid * 32 + i];
          uint32_t s = 8;
          if(b == '\n') { ty = (ty + 1) & 3u; at_start = true; have_q = false; }
          else {
            const bool first_of_line = at_start;
            if(at_start && (b != '\r' || a.min_qual)) {
              at_start = false;
              if(ty == 0) { s = SYM_BREAK; if(b != '@') atomicAdd(&a.T.stats[STAT_FORMAT_ERR], 1ull); }
              else if(ty == 2 && b != '+') atomicAdd(&a.T.stats[STAT_FORMAT_ERR], 1ull);
            }
            if(ty == 1 && a.min_qual) {
              // whole_sequence_parser.hpp:154-193 + mer_qual_iterator.hpp:64-92, 4-line records: the quality line is the
              // second line after this one, same column
              const long long g = g0 + i;
              if(!have_q) {
                long long sl = g;                    // start of this sequence line
                while(sl > -(long long)a.n_back && a.in[sl - 1] != '\n') --sl;
                long long e1 = g; while(e1 < (long long)a.n_look && a.in[e1] != '\n') ++e1;
                long long e2 = e1 + 1; while(e2 < (long long)a.n_look && a.in[e2] != '\n') ++e2;
                qoff = e2 + 1 - sl; have_q = true;
                if(e2 >= (long long)a.n_look) { atomicAdd(&a.T.stats[STAT_FORMAT_ERR], 1ull); have_q = false; }
                else if(first_of_line) {             // once per read: as many qualities as bases
                  long long e3 = e2 + 1; while(e3 < (long long)a.n_look && a.in[e3] != '\n') ++e3;
                  if(e3 - (e2 + 1) != e1 - sl) atomicAdd(&a.T.stats[STAT_FORMAT_ERR], 1ull);
                }
              }
              s = base_symbol(b);
              if(have_q) {                             // (a quality line shorter than its read is reported by the thread at the line start;
                const long long qp = g + qoff;          //  nobody reads past the text for it)
                if(qp >= (long long)a.n_look || (signed char)a.in[qp] < (signed char)a.min_qual) s = SYM_BREAK;
              }
            } else if(ty == 1) {
              if(b == '\r') { if(!cr_dropped(a.in, (uint64_t)(g0 + i), a.n_look)) s = SYM_BREAK; }
              else s = base_symbol(b);
            }
          }
          if(s != 8) { sy |= (uint64_t)(s & 3u) << (2 * cnt); bk |= (uint32_t)(s == SYM_BREAK) << cnt; ++cnt; }
        }
      }
    } else {
      uint32_t st = st_in;
#pragma unroll 1
      for(int i = vlo; i < vhi; ++i) {
        {
          const uint32_t b = sm.win[tid * 32 + i];
          uint32_t s = 8;   // 8 = nothing
          if(st == ST_H) { if(b == '\n') st = ST_L; }
          else if(b == '\n') st = ST_L;
          else if(st == ST_L) {
            if(b == '\r') { }
            else if(b == '>') { st = ST_H; s = SYM_BREAK; }
            else { st = ST_S; s = base_symbol(b); }
          } else {           // ST_S
            if(b == '\r') { if(!cr_dropped(a.in, (uint64_t)(g0 + i), a.n_look)) s = SYM_BREAK; }
            else s = base_symbol(b);
          }
          if(s != 8) { sy |= (uint64_t)(s & 3u) << (2 * cnt); bk |= (uint32_t)(s == SYM_BREAK) << cnt; ++cnt; }
        }
      }
    }
    uint32_t cinc = cnt;
#pragma unroll
    for(int o = 1; o < 32; o <<= 1) {
      uint32_t up = __shfl_up_sync(0xffffffffu, cinc, o);
      if(lane >= o) cinc += up;
    }
    if(lane == 31) sm.warp_cnt[warp] = cinc;
    if(tid == 0) sm.halo_break = 0;
    bsync(K1P_C);
    uint32_t woff;
    {
      uint32_t g = lane < NW ? sm.warp_cnt[lane] : 0u;
#pragma unroll
      for(int o = 1; o < NW; o <<= 1) {
        uint32_t up = __shfl_up_sync(0xffffffffu, g, o);
        if(lane >= o) g += up;
      }
      woff = __shfl_sync(0xffffffffu, g, warp ? warp - 1 : 0);
      if(warp == 0) woff = 0;
    }
    const uint32_t off = woff + cinc - cnt;
    if(tid == HALO / 32) sm.idx0 = off;                // symbols emitted by the halo bytes
    if(tid == NTH - 1) sm.nsym = off + cnt;
    if(tid < HALO / 32 && bk) sm.halo_break = 1;
    if(cnt) {
      // OR the symbols into the packed streams at stream position PRE + off
      const uint32_t pos = PREK + off;
      const uint32_t sh = (pos & 15u) * 2u;
      const uint32_t lo = (uint32_t)sy, hi = (uint32_t)(sy >> 32);
      const uint32_t x0 = lo << sh, x1 = __funnelshift_l(lo, hi, sh), x2 = __funnelshift_l(hi, 0u, sh);
      uint32_t* dst = sm.rev + (pos >> 4);
      if(x0) atomicOr(dst, x0);
      if(x1) atomicOr(dst + 1, x1);
      if(x2) atomicOr(dst + 2, x2);
      if(bk) {
        const uint32_t s2 = pos & 31u;
        const uint32_t y0 = bk << s2, y1 = __funnelshift_l(bk, 0u, s2);
        if(y0) atomicOr(sm.brk + (pos >> 5), y0);
        if(y1) atomicOr(sm.brk + (pos >> 5) + 1, y1);
      }
    }
    bsync(K1P_OR);
    // the window's bytes are dead from here on (the per-byte paths above read them from shared memory): fetch the next one
    { const uint64_t tn = t + gridDim.x; if(tn < a.n_tiles && tid == 0) issue(tn); }
    const uint32_t idx0 = sm.idx0, nsym = sm.nsym;

    // ---- phase D: the PRE symbols in front of the window (stream words 0 .. PW-1) ----
    if(warp == 0) {
      if(t == 0) {
        sm.pre[lane] = a.carry_in->sym[lane]; sm.pre[lane + 32] = a.carry_in->sym[lane + 32];
        if constexpr(PREK > 64) { sm.pre[lane + 64] = a.carry_in->sym[lane + 64]; sm.pre[lane + 96] = a.carry_in->sym[lane + 96]; }
      } else {
        sm.pre[lane] = SYM_BREAK; sm.pre[lane + 32] = SYM_BREAK;
        if constexpr(PREK > 64) { sm.pre[lane + 64] = SYM_BREAK; sm.pre[lane + 96] = SYM_BREAK; }
        __syncwarp();
        const bool in_seq = a.format == 1 ? (a.tile_state[t] == 1) : (a.tile_state[t] != ST_H);
        if(lane == 0 && in_seq && idx0 < k - 1 && !sm.halo_break) {
          // pathological input (very short lines / long runs of blank lines): exact slow path
          if(a.format == 1) backfill_fastq<PREK>(a.in, a.n_look, a.carry_in, h, PREK, sm.pre, a.min_qual, a.n_back);
          else backfill_symbols<PREK>(a.in, a.n_look, a.carry_in, h, -2, PREK, sm.pre, a.min_qual != 0);
        }
      }
      __syncwarp();
      if(lane < PREK / 16) {                                // one 32-bit word of 16 symbols per lane
        uint32_t x = 0;
        for(int i = 0; i < 16; ++i) x |= (uint32_t)(sm.pre[lane * 16 + i] & 3u) << (2 * i);
        sm.rev[lane] = x;
      } else if(lane < PREK / 16 + PREK / 32) {
        const int q = lane - PREK / 16;
        uint32_t x = 0;
        for(int i = 0; i < 32; ++i) x |= (uint32_t)(sm.pre[q * 32 + i] >= SYM_BREAK) << i;
        sm.brk[q] = x;
      }
    }
    bsync(K1P_D);

    // hand the parser state to the next batch
    if(t == a.n_tiles - 1 && warp == 1) {
      uint8_t* cs = a.carry_out->sym;
      // (FASTQ: the backfill reads the line that holds byte n - 1, so the batch has to end in a sequence line; one that ends
      // in a header, '+' or quality line hands over the stream, whose last reset is that header's or comes before the next)
      const bool not_seq = a.format == 1 ? (a.tile_state[t] != 1 || (sm.total_state & 3u) != 1u) : (a.tile_state[t] == ST_H);
      if(nsym >= (uint32_t)PREK || t == 0 || sm.halo_break || not_seq) {
#pragma unroll
        for(int q = 0; q < PREK / 32; ++q) {                // the last PREK symbols of the stream
          const uint32_t s = nsym + lane + 32 * q;
          const uint32_t code = (sm.rev[s >> 4] >> (2 * (s & 15u))) & 3u;
          cs[lane + 32 * q] = (uint8_t)(((sm.brk[s >> 5] >> (s & 31u)) & 1u) ? SYM_BREAK : code);
        }
      } else if(lane == 0) {
        if(a.format == 1) backfill_fastq<PREK>(a.in, a.n_look, a.carry_in, (long long)n, PREK, cs, a.min_qual, a.n_back);
        else backfill_symbols<PREK>(a.in, a.n_look, a.carry_in, (long long)n, -2, PREK, cs, a.min_qual != 0);
      }
      if(lane == 0) a.carry_out->state = a.format == 1 ? (sm.total_state | (a.in[n - 1] == '\n' ? 4u : 0u)) : sm.total_state;
    }

    // ---- phase E: thread c owns stream word PW + c: the k-mers ending at its 32 symbols ----
    const uint32_t n_words = (nsym + 31) / 32;
    // which of the 32 end positions of stream word PW + c carry a k-mer: inside [idx0, nsym), no reset among the last k symbols
    auto kmer_mask = [&](const uint32_t c) -> uint32_t {
      const uint32_t W = PW + c;
      const int lo_i = (int)idx0 - (int)(32 * c), hi_i = (int)nsym - (int)(32 * c);
      uint32_t vmask = low_mask32((uint32_t)(hi_i > 32 ? 32 : hi_i)) & ~low_mask32((uint32_t)(lo_i < 0 ? 0 : (lo_i > 32 ? 32 : lo_i)));
      if constexpr(KW == 4) {
        // k > 32: a reset inside the word kills every end position from it on; of the resets in the 128 positions in front
        // of the word only the last one matters, and it kills the end positions up to k - 1 past it
        const uint32_t b0 = sm.brk[W];
        if(b0) vmask &= low_mask32(__ffs(b0) - 1);
#pragma unroll
        for(int d = 1; d <= 4; ++d) {
          const uint32_t bd = sm.brk[W - d];
          if(bd) {
            const int last = (31 - __clz(bd)) - 32 * d;              // relative to the word's first position (< 0)
            if(last + (int)k > 0) vmask &= ~low_mask32((uint32_t)min(last + (int)k, 32));
            break;
          }
        }
      } else {
        // resets in the 96 symbols ending with this word (k <= 64): dilate by k-1 positions
        uint64_t b_lo = ((uint64_t)sm.brk[W] << 32) | sm.brk[W - 1];           // positions 32(W-1) .. 32W+31
        uint32_t b_pp = KW == 2 ? sm.brk[W - 2] : 0u;
        if(b_lo | b_pp) {
          // bit (32 + i) of `d` = some reset in (i-k, i]
          uint64_t x = b_lo; uint32_t xp = b_pp;   // 96-bit value xp : x ... handled as: shift left with carry from xp
          uint32_t span = 1;
          // doubling: after the loop x covers `span` positions
          while(span * 2 <= k) {
            const uint64_t carry = span >= 32 ? ((uint64_t)xp << (span - 32)) : ((uint64_t)xp >> (32 - span));
            const uint32_t xp2 = span >= 32 ? 0u : (xp << span);
            x |= (x << span) | carry; xp |= xp2;
            span *= 2;
          }
          if(span < k) {
            const uint32_t r = k - span;
            const uint64_t carry = r >= 32 ? ((uint64_t)xp << (r - 32)) : ((uint64_t)xp >> (32 - r));
            x |= (x << r) | carry;
          }
          vmask &= ~(uint32_t)(x >> 32);
        }
      }
      return vmask;
    };
    // MODE 3: the rank of this thread's first k-mer in the window (exclusive scan of the popcounts of the masks; the window
    // holds at most NTH stream words, so thread c owns word c); the window's count goes to q_cnt[t]
    uint32_t q_rank = 0;
    if constexpr(MODE == 3) {
      const uint32_t pc = (uint32_t)tid < n_words ? __popc(kmer_mask(tid)) : 0u;
      uint32_t qinc = pc;
#pragma unroll
      for(int o = 1; o < 32; o <<= 1) {
        const uint32_t up = __shfl_up_sync(0xffffffffu, qinc, o);
        if(lane >= o) qinc += up;
      }
      if(lane == 31) sm.warp_cnt[warp] = qinc;
      __syncthreads();
      uint32_t g = lane < NW ? sm.warp_cnt[lane] : 0u;
#pragma unroll
      for(int o = 1; o < NW; o <<= 1) {
        const uint32_t up = __shfl_up_sync(0xffffffffu, g, o);
        if(lane >= o) g += up;
      }
      const uint32_t wo = warp ? __shfl_sync(0xffffffffu, g, warp - 1) : 0u;
      q_rank = wo + qinc - pc;
      if(tid == NTH - 1) a.q_cnt[t] = q_rank + pc;
    }
    if constexpr(KW == 4) {
      // four-word keys (k = 65..128): MODE 0 (direct insertion), MODE 1 (keys bucketed by owning shard) and MODE 3 (query
      // extraction), one k-mer at a time.
      // Key word q holds bases k-1-32q-31 .. k-1-32q from the end; the forward k-mer ending at stream position e is the
      // pair reversal of the 32-symbol pieces ending at e, e-32, ...; its reverse complement is the complement of the
      // pieces starting at e-k+1, e-k+33, ... (symbol s sits at bits 2(s&31) of rev64[s>>5])
      auto piece = [&](const uint32_t s) -> uint64_t {        // the 32 symbols from stream position s on
        const uint32_t w = s >> 5, sh = 2 * (s & 31u);
        return sh ? ((rev64[w] >> sh) | (rev64[w + 1] << (64 - sh))) : rev64[w];
      };
      uint64_t kmask[4];
#pragma unroll
      for(int q = 0; q < 4; ++q) kmask[q] = kbits >= 64u * (q + 1) ? ~0ull : (kbits <= 64u * q ? 0ull : ((1ull << (kbits - 64 * q)) - 1ull));
      for(uint32_t c = tid; c < n_words; c += NTH) {
        const uint32_t vmask = kmer_mask(c);
        if(!vmask) continue;
        ls.kmers += __popc(vmask);
        for(uint32_t r = vmask; r; r &= r - 1) {
          const uint32_t j = __ffs(r) - 1;
          const uint32_t e = 32 * (PW + c) + j;              // stream position of the k-mer's last base
          uint64_t m[4], rc[4], key[4];
#pragma unroll
          for(int q = 0; q < 4; ++q) {
            m[q] = pair_reverse64(piece(e - 32 * q - 31)) & kmask[q];
            rc[q] = ~piece(e - k + 1 + 32 * q) & kmask[q];
          }
          bool use_rc = false;
          if(a.canonical) {
            int q = 3;
            while(q > 0 && rc[q] == m[q]) --q;
            use_rc = rc[q] < m[q];
          }
#pragma unroll
          for(int q = 0; q < 4; ++q) key[q] = use_rc ? rc[q] : m[q];
          if constexpr(MODE == 3) {
            const uint64_t at = (uint64_t)t * a.q_tile_cap + q_rank + __popc(vmask & low_mask32(j));
#pragma unroll
            for(int q = 0; q < 4; ++q) a.q_keys[at * 4 + q] = key[q];
          } else if constexpr(MODE == 1) {
            // the owner's bucket, as for k <= 64: one atomic per group of lanes with the same owner, then 32 bytes per key
            // in two 16-byte stores (the host checks that the buckets are 16-byte aligned)
            const uint64_t pos = gf2_hash<4>(lut, key, (int)a.nbytes);
            const uint32_t owner = a.shard_bits ? (uint32_t)(pos >> (a.T.lsize - a.shard_bits)) : 0u;
            const uint32_t peers = __match_any_sync(__activemask(), owner);
            const uint32_t leader = __ffs(peers) - 1;
            unsigned long long at = 0;
            if((uint32_t)lane == leader) at = atomicAdd(&a.route_counts[owner], (unsigned long long)__popc(peers));
            at = __shfl_sync(peers, at, leader) + __popc(peers & ((1u << lane) - 1u));
            if(at < a.route_cap) {
              ulonglong2* dst = reinterpret_cast<ulonglong2*>(a.route_keys + ((uint64_t)owner * a.route_cap + at) * 4);
              dst[0] = make_ulonglong2(key[0], key[1]);
              dst[1] = make_ulonglong2(key[2], key[3]);
            } else atomicAdd(&a.T.stats[STAT_ROUTE_DROPPED], 1ull);
          } else {
            const uint64_t pos = gf2_hash<4>(lut, key, (int)a.nbytes);
            if(table_add<4, SB>(a.T, key, pos, 1, ls)) ls.inserted++;
            else { ls.failed++; record_failure<4>(a.T, key, 1); }
          }
        }
      }
    } else {
    // (FAST: every thread makes exactly one trip, with an empty mask if it owns no word -- the ring passes below are block-wide)
    for(uint32_t c = tid; c < (FAST ? (uint32_t)NTH : n_words); c += NTH) {
      const uint32_t W = PW + c;
      uint32_t vmask = kmer_mask(c);
      if(c >= n_words) vmask = 0;
      if(!FAST && !vmask) continue;
      ls.kmers += __popc(vmask);
      // forward strand: pair-reversed words (first base most significant), reverse strand: the words as they are
      const uint64_t R0 = rev64[W], R1 = rev64[W - 1], R2 = KW == 2 ? rev64[W - 2] : 0ull;
      const uint64_t F0 = pair_reverse64(R0), F1 = pair_reverse64(R1), F2 = KW == 2 ? pair_reverse64(R2) : 0ull;
#pragma unroll 1
      for(int o = 0; o < 4; ++o) {
        const uint32_t vm8 = (vmask >> (8 * o)) & 0xFFu;
        if(!FAST && !vm8) continue;
        // X = forward words shifted so that end symbol 8o+7 sits at bits 0..1; Y = reverse words shifted so that the
        // first symbol of the k-mer ending at symbol 8o sits at bits 0..1
        const uint32_t fs = 48 - 16 * o;                   // 62 - 2(8o+7)
        uint64_t X0, X1, X2 = 0;                           // 192-bit window of the forward stream >> fs (low words)
        X0 = fs ? ((F0 >> fs) | (F1 << (64 - fs))) : F0;
        X1 = fs ? ((F1 >> fs) | (F2 << (64 - fs))) : F1;
        if(KW == 2) X2 = F2 >> fs;
        // reverse: stream position of the first symbol = 32(W) + 8o - (k-1), relative to word W-2 (KW=2) or W-1 (KW=1)
        uint64_t Y0, Y1, Y2 = 0;
        {
          const uint32_t q = (KW == 2 ? 64u : 32u) + 8u * o + 1u - k;      // symbols to drop from the bottom (>= 1)
          const uint32_t s = 2 * q;
          // value = R0:R1(:R2) with the oldest word lowest
          uint64_t v0 = KW == 2 ? R2 : R1, v1 = KW == 2 ? R1 : R0, v2 = KW == 2 ? R0 : 0ull;
          const uint32_t ws = s >> 6, bs = s & 63u;
          if(ws == 1) { v0 = v1; v1 = v2; v2 = 0; }
          else if(ws == 2) { v0 = v2; v1 = 0; v2 = 0; }
          else if(ws >= 3) { v0 = 0; v1 = 0; v2 = 0; }
          Y0 = bs ? ((v0 >> bs) | (v1 << (64 - bs))) : v0;
          Y1 = bs ? ((v1 >> bs) | (v2 << (64 - bs))) : v1;
          if(KW == 2) Y2 = bs ? (v2 >> bs) : v2;
        }
        // canonical (or forward) k-mer ending at symbol 8o+j
        auto kmer_at = [&](const int j, uint64_t (&key)[KW]) {
          uint64_t m[KW], rc[KW];
          const int ms = 14 - 2 * j;                       // forward: end symbol 8o+j
          const int rs = 2 * j;                            // reverse: first symbol moves up by j
          m[0]  = (ms ? ((X0 >> ms) | (X1 << (64 - ms))) : X0);
          rc[0] = ~(rs ? ((Y0 >> rs) | (Y1 << (64 - rs))) : Y0);
          if(KW == 1) { m[0] &= kmask_lo; rc[0] &= kmask_lo; }
          else {
            m[KW - 1]  = (ms ? ((X1 >> ms) | (X2 << (64 - ms))) : X1) & kmask_hi;
            rc[KW - 1] = ~(rs ? ((Y1 >> rs) | (Y2 << (64 - rs))) : Y1) & kmask_hi;
          }
          bool use_rc = false;
          if(a.canonical) {
            if(KW == 1) use_rc = rc[0] < m[0];
            else use_rc = (rc[KW - 1] < m[KW - 1]) || (rc[KW - 1] == m[KW - 1] && rc[0] < m[0]);
          }
#pragma unroll
          for(int q = 0; q < KW; ++q) key[q] = use_rc ? rc[q] : m[q];
        };
        if constexpr(FAST) {
          // a record into its region's ring (slot numbers are handed out by one shared-memory atomic on the packed counter);
          // a ring or a chunk that is full sends the k-mer to the spill list, the ring pass hands the slot out again
          auto ring_append = [&](const uint32_t p, const uint32_t rec, const int j) {
            const uint32_t v = atomicAdd(&st_cnt[p], 1u);
            const uint32_t slot = v & 0xFFFFu, fl = v >> 16;
            if(slot - fl < rlen && slot < pd.chunk_recs) ring[ring_word(p, slot)] = rec;
            else if(pd.by_owner) atomicAdd(&a.T.stats[STAT_ROUTE_DROPPED], 1ull);   // sharded send side: another shard's k-mer cannot be spilled here
            else {
              uint64_t key[KW];
              kmer_at(j, key);
              const uint64_t pos = ((uint64_t)p << f_rgb) | (rec >> f_hb);
              spill_record<KW, SB>(a.T, pd.spill_keys, pd.spill_counts, pd.spill_n, pd.spill_cap, key[0], key[KW - 1], pos, pd.lazy_win);
            }
          };
#pragma unroll
          for(int hf = 0; hf < 8; hf += SG) {
            const uint32_t vm4 = (vm8 >> hf) & ((1u << SG) - 1u);
            if(vm4) {          // (the host launches the FAST form only without a Bloom filter in front of the table)
              // two passes over the SG k-mers so that the shared-memory round trips overlap: keys, hashes and records (4 SG
              // independent table loads in flight), then the slot reservations and the ring stores
              uint32_t P[SG], R[SG];
#if JF_K1_PROF
              const long long prof_h = clock64();
#endif
#pragma unroll
              for(int jj = 0; jj < SG; ++jj) {
                const int j = hf + jj;
                // (computed for the masked-out positions as well: no branch per k-mer; kbits <= 44 keeps every table index in range)
                uint64_t key[KW];
                kmer_at(j, key);
                const uint32_t klo = (uint32_t)key[0], khi = (uint32_t)(key[0] >> 32);
                const uint32_t h32 = lut32[klo & 2047u] ^ lut32[2048 + ((klo >> 11) & 2047u)] ^
                                     lut32[4096 + (__funnelshift_r(klo, khi, 22) & 2047u)] ^ lut32[6144 + ((khi >> 1) & 2047u)];
                uint32_t ext = 0;                 // position bits 32.. : one parity row each (two for a table of 2^34 slots)
#pragma unroll
                for(int r = 0; r < NPR; ++r) ext |= (__popc((klo & (uint32_t)a.prow[r]) ^ (khi & (uint32_t)(a.prow[r] >> 32))) & 1u) << r;
                P[jj] = (h32 >> f_rgb) | (ext << (32 - f_rgb));                       // region
                R[jj] = ((h32 & f_relmask) << f_hb) | (uint32_t)(key[0] >> f_lsz);    // (position in the region, explicit key bits)
              }
#if JF_K1_PROF
              if(lane == 0) prof_w[warp][2 * K1P_SEGS] += clock64() - prof_h;
#endif
#pragma unroll
              for(int jj = 0; jj < SG; ++jj) if((vm4 >> jj) & 1u) ring_append(P[jj], R[jj], hf + jj);
            }
            // single-GPU counting: one ring pass per 8 k-mers per thread.  A ring of 32 then takes Poisson(8) records per pass on
            // top of at most 7 of an incomplete group and overflows in about 1e-6 of the region-passes, into the exact spill list.
            // The sharded send side cannot spill another shard's k-mer, so it keeps a pass per SG k-mers.
            if(hf + SG < 8 && !pd.by_owner) continue;
            bsync(K1P_APPEND);
            flush_rings(false);
            bsync(K1P_PASS);
          }
        } else {
#pragma unroll
        for(int j = 0; j < 8; ++j) {
          if(!((vm8 >> j) & 1u)) continue;
          uint64_t key[KW];
          kmer_at(j, key);
          if constexpr(MODE == 3) {        // input order: the k-mers ending in front of this one in the window come first
            const uint64_t at = (uint64_t)t * a.q_tile_cap + q_rank + __popc(vmask & low_mask32(8u * o + j));
#pragma unroll
            for(int q = 0; q < KW; ++q) a.q_keys[at * KW + q] = key[q];
            continue;
          }
          if(a.bloom.mode) {
            const uint64_t h1 = gf2_hash<KW>(bl1, key, (int)a.nbytes), h2 = gf2_hash<KW>(bl2, key, (int)a.nbytes);
            if(a.bloom.mode == BLOOM_COUNT) { bloom_count(a.bloom, h1, h2); ls.inserted++; continue; }   // `jellyfish bc`: no table
            if(a.bloom.mode == BLOOM_FILTER ? !bloom_test_and_set(a.bloom, h1, h2) : !bloom_check(a.bloom, h1, h2)) continue;
          }
          uint64_t pos;
          if(KW == 1 && a.hash_fast) {
            const uint64_t kk = key[0];
            uint32_t h32 = lut32[(uint32_t)kk & 2047u] ^ lut32[2048 + ((uint32_t)(kk >> 11) & 2047u)] ^
                           lut32[4096 + ((uint32_t)(kk >> 22) & 2047u)] ^ lut32[6144 + (uint32_t)(kk >> 33)];
            pos = h32;
            for(uint32_t jb = 0; jb < a.n_prow; ++jb) pos |= (uint64_t)(__popcll(kk & a.prow[jb]) & 1) << (32 + jb);
          } else pos = gf2_hash<KW>(lut, key, (int)a.nbytes);
          if(MODE == 0) {
            if(table_add<KW, SB>(a.T, key, pos, 1, ls)) ls.inserted++;
            else { ls.failed++; record_failure<KW>(a.T, key, 1); }
          } else if(MODE == 1) {
            const uint32_t owner = a.shard_bits ? (uint32_t)(pos >> (a.T.lsize - a.shard_bits)) : 0u;
            const uint32_t peers = __match_any_sync(__activemask(), owner);
            const uint32_t leader = __ffs(peers) - 1;
            unsigned long long at = 0;
            if((uint32_t)lane == leader) at = atomicAdd(&a.route_counts[owner], (unsigned long long)__popc(peers));
            at = __shfl_sync(peers, at, leader) + __popc(peers & ((1u << lane) - 1u));
            if(at < a.route_cap) {
#pragma unroll
              for(int q = 0; q < KW; ++q) a.route_keys[((uint64_t)owner * a.route_cap + at) * KW + q] = key[q];
            } else atomicAdd(&a.T.stats[STAT_ROUTE_DROPPED], 1ull);
          } else {
            // record = (position inside the region << hb) | explicit key bits
            const uint64_t lpos = pos & a.T.local_mask;
            const uint32_t p = (uint32_t)(lpos >> pd.region_bits);
            const uint64_t rel = lpos & ((1ull << pd.region_bits) - 1ull);
            const u128 rec = rec_make(key_high<KW>(key, a.T.lsize), rel, a.T.fbits - a.T.rbits);
            const uint32_t slot = atomicAdd(&st_cnt[p], 1u);
            if(slot < pd.chunk_recs) store_rec(pd.pool + (size_t)st_chunk[p] * CHUNK_BYTES, pd.rec_bytes, slot, rec);
            else spill_record<KW, SB>(a.T, pd.spill_keys, pd.spill_counts, pd.spill_n, pd.spill_cap, key[0], key[KW - 1], pos, pd.lazy_win);    // this region's chunk filled up within one window (skewed input)
          }
        }
        }
      }
    }
    }
    bsync(K1P_EEND);     // all reads of the streams done
    // clear the stream words this window used (the next window ORs into them) and roll full chunks over
    for(uint32_t i = tid; i < 2 * (n_words + PW) + 3; i += NTH) sm.rev[i] = 0;
    for(uint32_t i = tid; i < n_words + PW + 2; i += NTH) sm.brk[i] = 0;
    if(MODE == 2 && !FAST) for(uint32_t p = tid; p < pd.P; p += NTH) roll_chunk(pd, p, a.T.stats, st_chunk, st_cnt);
    bsync(K1P_WEND);
  }
#if JF_K1_PROF
  if constexpr(PROF) {
    if(lane == 0) {
      prof_w[warp][2 * K1P_SEGS + 1] = clock64() - prof_start;
      for(int i = 0; i < 2 * K1P_SEGS + 2; ++i) atomicAdd(&k1_prof_acc[i], prof_w[warp][i]);
    }
    if(tid == 0) {
      atomicAdd(&k1_prof_acc[2 * K1P_SEGS + 2], (unsigned long long)(blockIdx.x < a.n_tiles ? (a.n_tiles - blockIdx.x + gridDim.x - 1) / gridDim.x : 0));
      atomicAdd(&k1_prof_acc[2 * K1P_SEGS + 3], 1ull);
    }
  }
#endif
  if(MODE == 2) {          // keep the open chunks for the next launch
    if(FAST) { flush_rings(true); __syncthreads(); }
    for(uint32_t p = tid; p < pd.P; p += NTH) { my_chunk[p] = st_chunk[p]; my_fill[p] = min(FAST ? (st_cnt[p] & 0xFFFFu) : st_cnt[p], pd.chunk_recs); }
    if(own_arena && tid == 0) pd.pool_next[blockIdx.x] = *arena_next;
  }

  // ---- statistics: one atomic per counter per CTA (a query leaves them alone) ----
  if constexpr(MODE == 3) return;
  unsigned long long v[4] = { ls.kmers, ls.inserted, ls.distinct, ls.reprobes };
#pragma unroll
  for(int q = 0; q < 4; ++q) {
#pragma unroll
    for(int o = 16; o; o >>= 1) v[q] += __shfl_xor_sync(0xffffffffu, v[q], o);
  }
  if(lane == 0) { sm.part[warp][0] = v[0]; sm.part[warp][1] = v[1]; sm.part[warp][2] = v[2]; sm.part[warp][3] = v[3]; }
  __syncthreads();
  if(tid < 4) {
    unsigned long long s = 0;
    for(int i = 0; i < NW; ++i) s += sm.part[i][tid];
    const int which = tid == 0 ? STAT_KMERS : tid == 1 ? STAT_INSERTED : tid == 2 ? STAT_DISTINCT : STAT_REPROBES;
    if(s) atomicAdd(&a.T.stats[which], s);
  }
}

}  // namespace jfk
#endif
