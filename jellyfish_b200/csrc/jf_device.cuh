// jf_device.cuh -- device-side building blocks of the H100 k-mer counting engine.
//
// Data layout in HBM (see DESIGN.md):
//  * input text: raw FASTA bytes, processed in windows of WIN = HALO + TILE bytes that a
//    CTA stages into shared memory with one TMA bulk copy (cp.async.bulk) per window;
//  * table: ONE array of fixed-width slots (32, 64 or 128 bit), slot = [counter | key field],
//    key field = (key bits [l,2k) << rbits) | (reprobe+1)  -- the quotienting of the
//    reference (large_hash_array.hpp:519-533: "MSB of key | reprobe"), 0 = empty;
//    the counter lives in the HIGH bits so a carry out of it falls off the word and can
//    never corrupt the key field; carries are counted exactly in a small side table;
//  * probe i of a key with hash position pos goes to pos + i(i+1)/2 (lib/storage.cc:13-41),
//    i <= max_reprobe; shards do not wrap, they own an overflow margin instead.
#ifndef JF_DEVICE_CUH
#define JF_DEVICE_CUH
#include <stdint.h>
#include <cuda_runtime.h>
#include <type_traits>

namespace jfk {

constexpr int HALO  = 256;          // bytes of the previous tile staged again in front of a tile
constexpr int PRE   = 64;           // symbol slots kept in front of a window (>= k-1) for k <= 64
constexpr int PRE_WIDE = 128;       // the same for four-word keys (k <= 128)

enum { ST_H = 0, ST_S = 1, ST_L = 2 };   // inside header line / inside sequence line / at line start
constexpr uint32_t SYM_BREAK = 4;        // symbols 0..3 = A,C,G,T ; 4 = window reset

// stats block indices
enum { STAT_KMERS = 0, STAT_INSERTED, STAT_DISTINCT, STAT_REPROBES, STAT_OVERFLOWED,
       STAT_FAILED, STAT_FAIL_DROPPED, STAT_OVF_FULL, STAT_ROUTE_DROPPED, STAT_MAXCOUNT, STAT_POOL_FULL, STAT_FORMAT_ERR, STAT_N };

struct Carry {               // parser state handed from one batch to the next (device resident)
  uint32_t state;            // ST_* after the last byte of the previous batch
  uint32_t pad;
  uint8_t  sym[PRE_WIDE];    // last PRE (PRE_WIDE for four-word keys) symbols emitted (left-padded with SYM_BREAK)
};

struct TableDev {
  void*     slots;
  uint64_t  local_mask;      // (slots owned by this shard) - 1
  uint32_t  local_lsize;     // log2 of owned slots
  uint32_t  lsize;           // log2 of the GLOBAL table size (header "size")
  uint32_t  shard_index;
  uint32_t  kbits;           // 2k
  uint32_t  rbits;           // width of the reprobe field
  uint32_t  fbits;           // width of the key field  = max(2k - lsize, 0) + rbits
  uint32_t  max_reprobe;
  uint32_t  op;              // 0 COUNT (add), 1 PRIME (insert with count 0), 2 UPDATE (add only to keys already present)
  unsigned long long* ovf_keys;    // side table for counter carries: slot index + 1
  unsigned long long* ovf_vals;    //   number of carries (units of 2^cbits)
  uint64_t  ovf_mask;
  unsigned long long* stats;       // STAT_N counters
  uint64_t* fail_keys;             // keys that found no slot (reprobe limit hit)
  uint64_t* fail_counts;
  uint64_t  fail_cap;
};

// Bloom structures in front of the table (count_main.cc:99-131): `--bf-size` one-pass prefilter (bloom_filter.hpp:42-69),
// `jellyfish bc` Bloom counter (bloom_counter2.hpp:56-107) and `count --bc` filtering by a loaded counter.
// Positions of a key: base = h1 mod m, inc = h2 mod m, position i = (base + i*inc) mod m (h1, h2 = two 64-row GF(2)
// products of the key, mer_dna_bloom_counter.hpp:20-34).
enum { BLOOM_NONE = 0, BLOOM_FILTER = 1, BLOOM_COUNT = 2, BLOOM_CHECK = 3 };
struct BloomDev {
  uint32_t mode;               // BLOOM_*
  uint32_t k;                  // number of positions per key
  uint64_t m;                  // number of positions
  uint64_t inv;                // floor(2^64 / m)
  uint32_t* bits;              // FILTER: 1 bit per position; COUNT: 2 bits per position ("hit once", "hit twice");
                               // CHECK: 1 bit per position (the base-3 digit of the loaded counter is 2)
  uint32_t* locks;             // FILTER: per-key serialisation (2^lock_bits words)
  uint32_t lock_mask;
  uint32_t pad;
  const uint64_t* lut1;        // byte tables of the two 64-row matrices (global memory; staged in shared memory by K1)
  const uint64_t* lut2;
};

struct u128 { uint64_t lo, hi; };

__host__ __device__ __forceinline__ uint64_t tri(uint32_t i) { return (uint64_t)i * (i + 1) / 2; }

// ---------------------------------------------------------------------------------------
// PTX wrappers: mbarrier + 1-D TMA bulk copy (global -> shared), 128-bit CAS
// ---------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" :: "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile("{\n\t.reg .pred p;\n\t"
               "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
               "selp.u32 %0, 1, 0, p;\n\t}"
               : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  while(!mbar_try_wait(bar, parity)) { }
}
// TMA 1-D bulk copy: dst (shared, 16B aligned) <- src (global, 16B aligned), bytes % 16 == 0
__device__ __forceinline__ void tma_load_1d(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               :: "r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
// TMA 1-D bulk store: dst (global, 16B aligned) <- src (shared, 16B aligned), bytes % 16 == 0; completion is tracked per
// thread by bulk groups
__device__ __forceinline__ void tma_store_1d(void* dst, const void* src, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" :: "l"(dst), "r"(smem_u32(src)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tma_commit_group() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// all bulk groups of this thread have finished READING their shared-memory source
__device__ __forceinline__ void tma_wait_group_read0() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
// ... have completed (writes visible)
__device__ __forceinline__ void tma_wait_group0() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

__device__ __forceinline__ u128 atomic_cas_128(void* addr, u128 cmp, u128 val) {
  u128 old;
  asm volatile("{\n\t.reg .b128 c, s, d;\n\t"
               "mov.b128 c, {%2, %3};\n\t"
               "mov.b128 s, {%4, %5};\n\t"
               "atom.global.relaxed.gpu.cas.b128 d, [%6], c, s;\n\t"
               "mov.b128 {%0, %1}, d;\n\t}"
               : "=l"(old.lo), "=l"(old.hi)
               : "l"(cmp.lo), "l"(cmp.hi), "l"(val.lo), "l"(val.hi), "l"(addr) : "memory");
  return old;
}
__device__ __forceinline__ u128 load_128(const void* addr) {
  u128 v;
  asm volatile("ld.global.relaxed.gpu.v2.u64 {%0, %1}, [%2];" : "=l"(v.lo), "=l"(v.hi) : "l"(addr) : "memory");
  return v;
}

// ---------------------------------------------------------------------------------------
// base codes: reference mer_dna.hpp:38-55 -- A,a=0 C,c=1 G,g=2 T,t=3, everything else resets
// ---------------------------------------------------------------------------------------
__host__ __device__ __forceinline__ uint32_t base_symbol(uint32_t b) {
  uint32_t u = b & 0xDFu;                       // fold case
  uint32_t x = (b >> 1) & 3u;                   // A->0 C->1 G->3 T->2
  uint32_t code = x ^ (x >> 1);                 // A->0 C->1 G->2 T->3
  bool ok = (u == 'A') | (u == 'C') | (u == 'G') | (u == 'T');
  return ok ? code : SYM_BREAK;
}

// ---------------------------------------------------------------------------------------
// GF(2) hash through byte-indexed tables held in shared memory
// (rectangular_binary_matrix.hpp:223-261: XOR of columns[c-1-i] over the set bits i).
// lut[b*256 + v] = XOR of the columns selected by byte value v at byte position b.
// ---------------------------------------------------------------------------------------
template<int KW>
__device__ __forceinline__ uint64_t gf2_hash(const uint64_t* __restrict__ lut, const uint64_t (&key)[KW], int nbytes) {
  uint64_t h = 0;
#pragma unroll
  for(int b = 0; b < 8 * KW; ++b) {
    if(b < nbytes) {
      uint32_t v = (uint32_t)(key[b >> 3] >> ((b & 7) * 8)) & 0xFFu;
      h ^= lut[b * 256 + v];
    }
  }
  return h;
}

// key >> lsize for a KW-word key (the bits that are stored explicitly)
template<int KW>
__device__ __forceinline__ u128 key_high(const uint64_t (&key)[KW], uint32_t lsize) {
  u128 r;
  if(KW == 1) {
    r.lo = lsize >= 64 ? 0 : key[0] >> lsize;
    r.hi = 0;
  } else {
    uint64_t k0 = key[0], k1 = key[KW - 1];
    if(lsize == 0)       { r.lo = k0; r.hi = k1; }
    else if(lsize < 64)  { r.lo = (k0 >> lsize) | (k1 << (64 - lsize)); r.hi = k1 >> lsize; }
    else                 { r.lo = lsize >= 128 ? 0 : k1 >> (lsize - 64); r.hi = 0; }
  }
  return r;
}

// global position of a slot of this shard: shard bits : local position
__device__ __forceinline__ uint64_t global_pos(const TableDev& T, uint64_t local_pos) {
  return ((uint64_t)T.shard_index << T.local_lsize) | local_pos;
}

// the inverse of key_high and the hash: the key whose explicit bits are `high` and whose hash is the global position
// `gpos`.  The low lsize key bits are the inverse matrix times [high : gpos] (large_hash_iterator.hpp:164-170;
// large_hash_array.hpp:851-858).
template<int KW>
__device__ __forceinline__ void key_from_position(const uint64_t* __restrict__ inv_lut, uint32_t nbytes, uint32_t lsize, u128 high,
                                                  uint64_t gpos, uint64_t (&key)[KW]) {
  uint64_t v[KW];
  v[0] = (lsize >= 64 ? 0 : (high.lo << lsize)) | gpos;
  if(KW == 2) v[KW - 1] = lsize ? ((high.hi << lsize) | (high.lo >> (64 - lsize))) : high.hi;
  const uint64_t low = gf2_hash<KW>(inv_lut, v, (int)nbytes);
  const uint64_t lmask = lsize >= 64 ? ~0ull : ((1ull << lsize) - 1ull);
#pragma unroll
  for(int q = 0; q < KW; ++q) key[q] = v[q];
  key[0] = (key[0] & ~lmask) | (low & lmask);
}

// ---------------------------------------------------------------------------------------
// Bloom filter / Bloom counter operations
// ---------------------------------------------------------------------------------------
__device__ __forceinline__ uint64_t bloom_mod(const BloomDev& B, uint64_t h) {
  uint64_t r = h - __umul64hi(h, B.inv) * B.m;         // quotient estimate is off by one at most
  while(r >= B.m) r -= B.m;
  return r;
}
// bloom_filter_base::insert__ (bloom_filter.hpp:42-69): set the k bits, return whether all of them were set before.
// Threads holding the SAME key are serialised through a small lock table, so that of n simultaneous occurrences of a
// k-mer that is not in the filter yet exactly one is reported absent -- the sequential semantics of the reference
// (filter_bf, count_main.cc:122-133: the first occurrence is dropped, later ones are counted).
__device__ __forceinline__ bool bloom_test_and_set(const BloomDev& B, uint64_t h1, uint64_t h2) {
  uint64_t pos = bloom_mod(B, h1);
  const uint64_t inc = bloom_mod(B, h2);
  uint32_t* lock = B.locks + (((uint32_t)h1 ^ (uint32_t)(h1 >> 32) ^ (uint32_t)h2) & B.lock_mask);
  bool present = true, done = false;
  while(!done) {
    if(atomicCAS(lock, 0u, 1u) == 0u) {
      for(uint32_t i = 0; i < B.k; ++i) {
        const uint32_t bit = 1u << (pos & 31u);
        const uint32_t old = atomicOr(&B.bits[pos >> 5], bit);
        present = present && (old & bit);
        pos += inc; if(pos >= B.m) pos -= B.m;
      }
      __threadfence();
      atomicExch(lock, 0u);
      done = true;
    }
  }
  return present;
}
// bloom_counter2_base::insert__ (bloom_counter2.hpp:56-107): every position is a counter saturating at 2.  Held as two
// bits ("hit", "hit again"), so the final state -- min(2, number of hits) -- does not depend on the order of the hits.
__device__ __forceinline__ void bloom_count(const BloomDev& B, uint64_t h1, uint64_t h2) {
  uint64_t pos = bloom_mod(B, h1);
  const uint64_t inc = bloom_mod(B, h2);
  for(uint32_t i = 0; i < B.k; ++i) {
    const uint32_t sh = (uint32_t)(pos & 15u) * 2u;
    uint32_t* w = &B.bits[pos >> 4];
    const uint32_t old = atomicOr(w, 1u << sh);
    if((old >> sh) & 1u) atomicOr(w, 2u << sh);
    pos += inc; if(pos >= B.m) pos -= B.m;
  }
}
// filter_bc (count_main.cc:110-120): bloom_counter2_base::check__ > 1, i.e. every position holds the digit 2
__device__ __forceinline__ bool bloom_check(const BloomDev& B, uint64_t h1, uint64_t h2) {
  uint64_t pos = bloom_mod(B, h1);
  const uint64_t inc = bloom_mod(B, h2);
  for(uint32_t i = 0; i < B.k; ++i) {
    if(!((__ldg(&B.bits[pos >> 5]) >> (pos & 31u)) & 1u)) return false;
    pos += inc; if(pos >= B.m) pos -= B.m;
  }
  return true;
}

// ---------------------------------------------------------------------------------------
// counter-carry side table (exact counts beyond the in-slot counter field)
// ---------------------------------------------------------------------------------------
__device__ __forceinline__ void ovf_add(const TableDev& T, uint64_t slot_idx, uint64_t carries) {
  const unsigned long long tag = slot_idx + 1;
  uint64_t h = (slot_idx * 0x9E3779B97F4A7C15ull) >> 20;
  for(uint32_t i = 0; i < 4096; ++i) {
    uint64_t p = (h + i) & T.ovf_mask;
    unsigned long long old = atomicCAS(&T.ovf_keys[p], 0ull, tag);
    if(old == 0ull || old == tag) {
      atomicAdd(&T.ovf_vals[p], (unsigned long long)carries);
      atomicAdd(&T.stats[STAT_OVERFLOWED], 1ull);
      return;
    }
  }
  atomicAdd(&T.stats[STAT_OVF_FULL], 1ull);
}
__device__ __forceinline__ uint64_t ovf_get(const TableDev& T, uint64_t slot_idx) {
  const unsigned long long tag = slot_idx + 1;
  uint64_t h = (slot_idx * 0x9E3779B97F4A7C15ull) >> 20;
  for(uint32_t i = 0; i < 4096; ++i) {
    uint64_t p = (h + i) & T.ovf_mask;
    unsigned long long k = T.ovf_keys[p];
    if(k == tag) return T.ovf_vals[p];
    if(k == 0ull) return 0;
  }
  return 0;
}

// ---------------------------------------------------------------------------------------
// insert-or-increment: hash_counter::add -> array::add -> claim_key/add_val
// (hash_counter.hpp:91-115, large_hash_array.hpp:291-295,509-597,741-752) re-designed for
// fixed-width slots and hardware atomics.  Returns false when max_reprobe+1 probes found
// no slot ("hash full").  SB = slot width in bits.
// ---------------------------------------------------------------------------------------
struct LocalStats { uint32_t kmers, inserted, distinct, reprobes, failed; };

// the end of an inserting kernel: a warp's insertion statistics summed over the warp, one atomic per nonzero sum
__device__ __forceinline__ void flush_stats(unsigned long long* stats, unsigned long long inserted, unsigned long long distinct,
                                            unsigned long long reprobes) {
  unsigned long long v[3] = { inserted, distinct, reprobes };
#pragma unroll
  for(int q = 0; q < 3; ++q) {
#pragma unroll
    for(int o = 16; o; o >>= 1) v[q] += __shfl_xor_sync(0xffffffffu, v[q], o);
  }
  if((threadIdx.x & 31) == 0) {
    if(v[0]) atomicAdd(&stats[STAT_INSERTED], v[0]);
    if(v[1]) atomicAdd(&stats[STAT_DISTINCT], v[1]);
    if(v[2]) atomicAdd(&stats[STAT_REPROBES], v[2]);
  }
}

template<int SB> __device__ __forceinline__ bool slot_decode(const TableDev& T, uint64_t idx, u128& high, uint32_t& reprobe, uint64_t& count);

// add `count` to the counter field of an occupied slot (carry -> side table)
template<int SB>
__device__ __forceinline__ void slot_add(const TableDev& T, uint64_t idx, uint64_t count) {
  if(count == 0) return;
  const uint32_t fb = T.fbits;
  if(SB == 32) {
    const uint32_t cb = 32 - fb;
    const uint32_t c_lo = (uint32_t)(count & ((1ull << cb) - 1));
    uint64_t carry = count >> cb;
    if(c_lo) { uint32_t o2 = atomicAdd(&((uint32_t*)T.slots)[idx], c_lo << fb); carry += ((uint64_t)(o2 >> fb) + c_lo) >> cb; }
    if(carry) ovf_add(T, idx, carry);
  } else {
    const uint32_t fhi = SB == 128 ? (fb > 64 ? fb - 64 : 0) : fb;
    const uint32_t cb = 64 - fhi;
    const uint64_t c_lo = cb >= 64 ? count : (count & ((1ull << cb) - 1));
    uint64_t carry = cb >= 64 ? 0 : (count >> cb);
    unsigned long long* wp = SB == 128 ? ((unsigned long long*)T.slots + 2 * idx + 1) : ((unsigned long long*)T.slots + idx);
    if(c_lo) {
      unsigned long long o2 = atomicAdd(wp, (unsigned long long)(c_lo << fhi));
      uint64_t oc = o2 >> fhi, sum = oc + c_lo;
      if((cb < 64 && (sum >> cb)) || sum < oc) carry += 1;
    }
    if(carry) ovf_add(T, idx, carry);
  }
}

// UPDATE (array::update_add, large_hash_array.hpp:335-347): add only when the key is already there
template<int SB>
__device__ __forceinline__ bool table_update_hp(const TableDev& T, const uint64_t base, const u128 high, uint64_t count) {
  uint64_t idx = base;
  for(uint32_t i = 0; i <= T.max_reprobe; ++i) {
    u128 h2; uint32_t rp; uint64_t cnt;
    if(!slot_decode<SB>(T, idx, h2, rp, cnt)) return true;            // empty slot: the key is not in the table
    if(rp == i && h2.lo == high.lo && h2.hi == high.hi) { slot_add<SB>(T, idx, count); return true; }
    idx = base + tri(i + 1);
  }
  return true;
}

template<int SB>
__device__ __forceinline__ bool table_add_hp(const TableDev& T, const uint64_t base, const u128 high,
                                             uint64_t count, LocalStats& ls, const uint32_t first_probe = 0) {
  if(T.op == 2) return table_update_hp<SB>(T, base, high, count);
  if(T.op == 1) count = 0;                   // PRIME (array::set, large_hash_array.hpp:313-319): claim the key, add nothing
  const uint32_t rb = T.rbits, fb = T.fbits;
  uint64_t idx = base + (first_probe ? tri(first_probe) : 0);

  if(SB == 32) {
    const uint32_t cb = 32 - fb;
    const uint32_t fmask = (1u << fb) - 1u;
    const uint32_t c_lo = (uint32_t)(count & ((1ull << cb) - 1));
    const uint64_t c_hi = count >> cb;
    uint32_t* tab = (uint32_t*)T.slots;
    const uint32_t kf0 = (uint32_t)(high.lo << rb);
    for(uint32_t i = first_probe; i <= T.max_reprobe; ++i) {
      const uint32_t kf = kf0 | (i + 1);
      uint32_t old = atomicCAS(&tab[idx], 0u, kf | (c_lo << fb));
      if(old == 0u) { ls.distinct++; ls.reprobes += i; if(c_hi) ovf_add(T, idx, c_hi); return true; }
      if((old & fmask) == kf) {
        uint32_t o2 = atomicAdd(&tab[idx], c_lo << fb);
        uint64_t carry = (((uint64_t)(o2 >> fb) + c_lo) >> cb) + c_hi;
        if(carry) ovf_add(T, idx, carry);
        ls.reprobes += i;
        return true;
      }
      idx = base + tri(i + 1);
    }
    return false;
  } else if(SB == 64) {
    const uint32_t cb = 64 - fb;
    const uint64_t fmask = (1ull << fb) - 1ull;
    const uint64_t c_lo = cb >= 64 ? count : (count & ((1ull << cb) - 1));
    const uint64_t c_hi = cb >= 64 ? 0 : (count >> cb);
    unsigned long long* tab = (unsigned long long*)T.slots;
    const uint64_t kf0 = high.lo << rb;
    for(uint32_t i = first_probe; i <= T.max_reprobe; ++i) {
      const uint64_t kf = kf0 | (i + 1);
      unsigned long long old = atomicCAS(&tab[idx], 0ull, (unsigned long long)(kf | (c_lo << fb)));
      if(old == 0ull) { ls.distinct++; ls.reprobes += i; if(c_hi) ovf_add(T, idx, c_hi); return true; }
      if((old & fmask) == kf) {
        unsigned long long o2 = atomicAdd(&tab[idx], (unsigned long long)(c_lo << fb));
        // carry out of the counter field: (old counter + c_lo) >= 2^cb
        uint64_t oc = o2 >> fb, sum = oc + c_lo;
        uint64_t carry = ((cb < 64 && (sum >> cb)) || sum < oc ? 1 : 0) + c_hi;
        if(carry) ovf_add(T, idx, carry);
        ls.reprobes += i;
        return true;
      }
      idx = base + tri(i + 1);
    }
    return false;
  } else {  // 128-bit slots: lo = low 64 bits of the key field, hi = [counter | rest of key field]
    const uint32_t fhi = fb > 64 ? fb - 64 : 0;       // key-field bits living in the hi word
    const uint32_t cb = 64 - fhi;
    const uint64_t fmask_hi = fhi ? ((1ull << fhi) - 1ull) : 0ull;
    const uint64_t c_lo = cb >= 64 ? count : (count & ((1ull << cb) - 1));
    const uint64_t c_hi = cb >= 64 ? 0 : (count >> cb);
    u128* tab = (u128*)T.slots;
    // key field = (high << rb) | (i+1)  as a 128-bit value
    const uint64_t kf_lo0 = high.lo << rb;
    const uint64_t kf_hi  = rb ? ((high.hi << rb) | (high.lo >> (64 - rb))) : high.hi;
    for(uint32_t i = first_probe; i <= T.max_reprobe; ++i) {
      const uint64_t kf_lo = kf_lo0 | (i + 1);
      u128 want; want.lo = kf_lo; want.hi = kf_hi | (c_lo << fhi);
      u128 zero; zero.lo = 0; zero.hi = 0;
      u128 old = atomic_cas_128(&tab[idx], zero, want);
      if(old.lo == 0 && old.hi == 0) { ls.distinct++; ls.reprobes += i; if(c_hi) ovf_add(T, idx, c_hi); return true; }
      if(old.lo == kf_lo && (old.hi & fmask_hi) == kf_hi) {
        unsigned long long* hp = (unsigned long long*)&tab[idx] + 1;
        unsigned long long o2 = atomicAdd(hp, (unsigned long long)(c_lo << fhi));
        uint64_t oc = o2 >> fhi, sum = oc + c_lo;
        uint64_t carry = ((cb < 64 && (sum >> cb)) || sum < oc ? 1 : 0) + c_hi;
        if(carry) ovf_add(T, idx, carry);
        ls.reprobes += i;
        return true;
      }
      idx = base + tri(i + 1);
    }
    return false;
  }
}

// R insertions of count 1.  Round 1: the R first probes (CAS) are issued back to back so the
// R L2 round trips overlap.  Keys that lost their first slot then LOOK AHEAD: the next LOOK probe
// slots (offsets 1,3,6,10 -- at most 40 bytes away, i.e. the same or the next 32-byte sector)
// are read with plain L2 loads, all in flight together, and only the first slot that is empty or
// already holds the key is CASed.  A dependent chain of p CAS round trips becomes ~2.
// ok[r] = false -> hash full.
template<typename W>
__device__ __forceinline__ W ld_slot(const W* p) { return __ldcg(p); }

template<int SB, int R>
__device__ __forceinline__ void table_add_batch(const TableDev& T, const uint64_t (&base)[R], const u128 (&high)[R],
                                                const bool (&valid)[R], bool (&ok)[R], LocalStats& ls) {
  constexpr uint32_t LOOK = 4;
  const uint32_t rb = T.rbits, fb = T.fbits;
  if(T.op != 0) {
#pragma unroll
    for(int r = 0; r < R; ++r) ok[r] = valid[r] ? table_add_hp<SB>(T, base[r], high[r], 1, ls) : true;
    return;
  }
  if(SB == 32 || SB == 64) {
    typedef typename std::conditional<SB == 32, uint32_t, unsigned long long>::type W;
    W* tab = (W*)T.slots;
    const W fmask = (W)(((W)1 << fb) - 1), one = (W)1 << fb;
    const uint32_t cb = SB - fb;
    W old[R], kf0[R];
#pragma unroll
    for(int r = 0; r < R; ++r) {
      kf0[r] = (W)((W)high[r].lo << rb);
      old[r] = valid[r] ? atomicCAS(&tab[base[r]], (W)0, (W)(kf0[r] | 1u | one)) : (W)1;
    }
    uint32_t pending = 0;
#pragma unroll
    for(int r = 0; r < R; ++r) {
      ok[r] = true;
      if(!valid[r]) continue;
      if(old[r] == 0) ls.distinct++;
      else if((old[r] & fmask) == (W)(kf0[r] | 1u)) {
        W o2 = atomicAdd(&tab[base[r]], one);
        if(((((uint64_t)(o2 >> fb)) + 1) >> cb) != 0) ovf_add(T, base[r], 1);
      } else pending |= 1u << r;
    }
#pragma unroll
    for(int r = 0; r < R; ++r) {
      if(!((pending >> r) & 1u)) continue;
      bool done = false;
      for(uint32_t nxt = 1; !done; nxt += LOOK) {
        if(nxt > T.max_reprobe) { ok[r] = false; break; }
        // look ahead: LOOK probe slots, loads all in flight
        W seen[LOOK];
#pragma unroll
        for(uint32_t j = 0; j < LOOK; ++j) {
          const uint32_t i = nxt + j;
          seen[j] = i <= T.max_reprobe ? ld_slot(&tab[base[r] + tri(i)]) : (W)~(W)0;
        }
#pragma unroll
        for(uint32_t j = 0; j < LOOK; ++j) {
          const uint32_t i = nxt + j;
          if(done || i > T.max_reprobe) continue;
          const W kf = (W)(kf0[r] | (W)(i + 1));
          const W v = seen[j];
          if(v != 0 && (v & fmask) != kf) continue;            // occupied by another key: keep walking
          const uint64_t idx = base[r] + tri(i);
          W o = v;
          if(v == 0) o = atomicCAS(&tab[idx], (W)0, (W)(kf | one));
          if(o == 0) { ls.distinct++; ls.reprobes += i; done = true; }
          else if((o & fmask) == kf) {
            W o2 = atomicAdd(&tab[idx], one);
            if(((((uint64_t)(o2 >> fb)) + 1) >> cb) != 0) ovf_add(T, idx, 1);
            ls.reprobes += i; done = true;
          }
          // else: another key took this slot in the meantime: keep walking
        }
      }
    }
  } else {
#pragma unroll
    for(int r = 0; r < R; ++r) ok[r] = valid[r] ? table_add_hp<SB>(T, base[r], high[r], 1, ls) : true;
  }
}

// ---------------------------------------------------------------------------------------
// The wide slot form (SB_WIDE, four-word keys, k = 65..128).  A quotiented key field would be 2k - l bits, up to 255, so
// a slot holds the whole canonical key instead: 40 bytes = a 64-bit HEAD word
//     head = [counter (high 64 - fbits bits) | READY (bit rbits) | reprobe+1 (low rbits bits)],  0 = empty,
// followed by the four key words.  The key sits next to its head (one slot = five consecutive words), so a probe that
// finds a head with its own reprobe index reads the key from the same or the next 32-byte sector.
//
// Claim / publish.  An inserter CASes the head from 0 to "claimed, not ready, reprobe i" (reprobe+1 alone), stores the
// four key words, __threadfence(), then sets READY and adds its count with ONE atomicAdd.  A prober that meets a head
// with its own reprobe index but without READY spins on the head until READY shows, fences, then compares the full key.
// No deadlock: the only thread a waiter can wait on is the claimer of that slot, and between its CAS and its publishing
// atomic the claimer executes four stores and a fence -- it waits on nothing and takes no other slot.  (Independent
// thread scheduling, sm_70 and later, lets the claimer progress even when a waiter shares its warp.)  Ordering: the
// claimer's fence + atomic is a release pattern, the waiter's load of READY + fence an acquire pattern, so the key words
// are visible to it.  A head with another reprobe index belongs to another key (the same key always lands at the same
// probe index from the same base) and is skipped without reading the key.
// ---------------------------------------------------------------------------------------
constexpr int SB_WIDE = 320;

__device__ __forceinline__ unsigned long long* wide_slot(const TableDev& T, uint64_t idx) {
  return (unsigned long long*)T.slots + 5 * idx;
}
__device__ __forceinline__ uint64_t ld_relaxed_u64(const unsigned long long* p) {
  uint64_t v;
  asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
// the head of a slot whose reprobe index is ours, once its key is published
__device__ __forceinline__ uint64_t wide_wait_ready(const unsigned long long* s, uint64_t head, uint64_t ready) {
  while(!(head & ready)) head = ld_relaxed_u64(s);
  __threadfence();
  return head;
}
__device__ __forceinline__ bool wide_key_eq(const unsigned long long* s, const uint64_t (&key)[4]) {
  return ld_relaxed_u64(s + 1) == key[0] && ld_relaxed_u64(s + 2) == key[1] && ld_relaxed_u64(s + 3) == key[2] &&
         ld_relaxed_u64(s + 4) == key[3];
}
// add c_lo << fbits to the head of an occupied slot; a carry out of the counter field and c_hi go to the side table
__device__ __forceinline__ void wide_count(const TableDev& T, uint64_t idx, unsigned long long* s, uint64_t c_lo, uint64_t c_hi) {
  const uint32_t fb = T.fbits, cb = 64 - fb;
  uint64_t carry = c_hi;
  if(c_lo) {
    const uint64_t oc = (uint64_t)atomicAdd(s, (unsigned long long)(c_lo << fb)) >> fb;
    if((oc + c_lo) >> cb) carry += 1;
  }
  if(carry) ovf_add(T, idx, carry);
}

// array::add / set / update_add (large_hash_array.hpp:291-347) on the wide form: T.op as in table_add_hp
__device__ __forceinline__ bool wide_add(const TableDev& T, const uint64_t base, const uint64_t (&key)[4], uint64_t count, LocalStats& ls) {
  const uint32_t rb = T.rbits, fb = T.fbits, cb = 64 - fb;
  const uint64_t ready = 1ull << rb, rmask = ready - 1;
  if(T.op == 1) count = 0;                   // PRIME: claim the key, add nothing
  const uint64_t c_lo = count & ((1ull << cb) - 1), c_hi = count >> cb;
  uint64_t idx = base;
  for(uint32_t i = 0; i <= T.max_reprobe; ++i) {
    unsigned long long* s = wide_slot(T, idx);
    uint64_t head;
    if(T.op == 2) {                          // UPDATE: never claims; an empty slot ends the probe sequence
      head = ld_relaxed_u64(s);
      if(head == 0) return true;
    } else {
      head = atomicCAS(s, 0ull, (unsigned long long)(i + 1));
      if(head == 0) {
        s[1] = key[0]; s[2] = key[1]; s[3] = key[2]; s[4] = key[3];
        __threadfence();
        atomicAdd(s, (unsigned long long)(ready | (c_lo << fb)));
        if(c_hi) ovf_add(T, idx, c_hi);
        ls.distinct++; ls.reprobes += i;
        return true;
      }
    }
    if((head & rmask) == i + 1) {
      head = wide_wait_ready(s, head, ready);
      if(wide_key_eq(s, key)) {
        wide_count(T, idx, s, c_lo, c_hi);
        ls.reprobes += i;
        return true;
      }
    }
    idx = base + tri(i + 1);
  }
  return T.op == 2;                          // (an update of an absent key is not a failure)
}

// count of `key` in the wide form (array::get_val_for_key), without the carries; false when absent
__device__ __forceinline__ bool wide_find(const TableDev& T, const uint64_t base, const uint64_t (&key)[4], uint64_t& idx_out, uint64_t& cnt) {
  const uint64_t rmask = (1ull << T.rbits) - 1;
  uint64_t idx = base;
  for(uint32_t i = 0; i <= T.max_reprobe; ++i) {
    const unsigned long long* s = wide_slot(T, idx);
    const uint64_t head = s[0];
    if(head == 0) return false;
    if((head & rmask) == i + 1 && s[1] == key[0] && s[2] == key[1] && s[3] == key[2] && s[4] == key[3]) {
      idx_out = idx; cnt = head >> T.fbits;
      return true;
    }
    idx = base + tri(i + 1);
  }
  return false;
}

template<int KW, int SB>
__device__ __forceinline__ bool table_add(const TableDev& T, const uint64_t (&key)[KW], uint64_t pos_global,
                                          uint64_t count, LocalStats& ls) {
  if constexpr(SB == SB_WIDE) return wide_add(T, pos_global & T.local_mask, key, count, ls);
  else return table_add_hp<SB>(T, pos_global & T.local_mask, key_high<KW>(key, T.lsize), count, ls);
}

template<int KW>
__device__ __forceinline__ void record_failure(const TableDev& T, const uint64_t (&key)[KW], uint64_t count) {
  unsigned long long at = atomicAdd(&T.stats[STAT_FAILED], 1ull);
  if(at < T.fail_cap) {
#pragma unroll
    for(int w = 0; w < KW; ++w) T.fail_keys[at * KW + w] = key[w];
    T.fail_counts[at] = T.op == 1 ? 0 : count;          // a primed key is re-inserted with count 0 after a regrow
  } else {
    atomicAdd(&T.stats[STAT_FAIL_DROPPED], 1ull);
  }
}

// Decode one slot. Returns false when empty. Outputs the explicit key bits, the reprobe
// index (0-based) and the in-slot counter.
template<int SB>
__device__ __forceinline__ bool slot_decode(const TableDev& T, uint64_t idx, u128& high, uint32_t& reprobe, uint64_t& count) {
  const uint32_t rb = T.rbits, fb = T.fbits;
  const uint64_t rmask = (1ull << rb) - 1ull;
  if(SB == SB_WIDE) {        // (the key is read from the slot by the callers that need it)
    const uint64_t v = ((const uint64_t*)T.slots)[5 * idx];
    if(v == 0) return false;
    reprobe = (uint32_t)(v & rmask) - 1;
    high.lo = 0; high.hi = 0;
    count = v >> fb;
    return true;
  } else if(SB == 32) {
    uint32_t v = ((const uint32_t*)T.slots)[idx];
    if(v == 0) return false;
    uint32_t kf = v & ((1u << fb) - 1u);
    reprobe = (uint32_t)(kf & rmask) - 1;
    high.lo = kf >> rb; high.hi = 0;
    count = v >> fb;
    return true;
  } else if(SB == 64) {
    uint64_t v = ((const uint64_t*)T.slots)[idx];
    if(v == 0) return false;
    uint64_t kf = v & ((1ull << fb) - 1ull);
    reprobe = (uint32_t)(kf & rmask) - 1;
    high.lo = kf >> rb; high.hi = 0;
    count = fb >= 64 ? 0 : v >> fb;
    return true;
  } else {
    u128 v = ((const u128*)T.slots)[idx];
    if(v.lo == 0 && v.hi == 0) return false;
    const uint32_t fhi = fb > 64 ? fb - 64 : 0;
    uint64_t kf_hi = fhi ? (v.hi & ((1ull << fhi) - 1ull)) : 0;
    reprobe = (uint32_t)(v.lo & rmask) - 1;
    high.lo = rb ? ((v.lo >> rb) | (kf_hi << (64 - rb))) : v.lo;
    high.hi = kf_hi >> rb;
    count = v.hi >> fhi;
    return true;
  }
}

// width of the in-slot counter field
template<int SB>
__device__ __forceinline__ uint32_t slot_counter_bits(const TableDev& T) {
  return SB == SB_WIDE ? 64 - T.fbits : (SB == 128) ? (64 - (T.fbits > 64 ? T.fbits - 64 : 0)) : (SB - T.fbits);
}

// the count of slot `idx` whose counter field holds `cnt`, with the carries of the side table; saturates at 2^64-1 like a
// 64-bit counter would.  (The callers skip it while no counter has ever carried: STAT_OVERFLOWED == 0.)  Only a 128-bit
// slot can have a 64-bit counter field; a wide slot's is at most 62 bits (fbits >= 2).
template<int SB>
__device__ __forceinline__ uint64_t slot_full_count(const TableDev& T, uint64_t idx, uint64_t cnt) {
  const uint32_t cb = slot_counter_bits<SB>(T);
  const uint64_t carries = ovf_get(T, idx);
  if(carries) {
    if((SB != SB_WIDE && cb >= 64) || (carries >> (64 - cb)) != 0) cnt = ~0ull;
    else { const uint64_t add = carries << cb; cnt = (cnt + add < cnt) ? ~0ull : cnt + add; }
  }
  return cnt;
}

}  // namespace jfk
#endif
