// jf_dump.cuh -- K3/K4, the sorted dump without a global sort.
//
// The reference's sorted_dumper (sorted_dumper.hpp:57-101) walks the table with a heap of
// reprobes[max_reprobe] entries because a key sits at most that many slots above its ORIGINAL
// position (large_hash_array.hpp:851-854).  The same bound makes the order a LOCAL property here:
// the records whose original position lies in [a, a + TP) all sit in the slots [a, a + TP + margin),
// so one CTA can produce that piece of the output on its own:
//   dump_count_kernel  per tile of TP positions: how many records it will emit (after the -L/-U filter);
//   dump_scan_kernel   exclusive scan of the tile counts of one segment (one CTA);
//   dump_emit_kernel   per tile: counting sort of the tile's records by original position in shared
//                      memory (positions are nearly unique: a bucket holds the handful of keys that hash to
//                      the same position, ordered by their explicit key bits with an insertion sort), then
//                      the record bytes -- ceil(2k/8) key bytes, out_counter_len count bytes
//                      (binary_dumper.hpp:36-40) -- staged in shared memory and written with coalesced stores.
// The table is read twice (plus L2 hits); nothing is sorted globally.
#ifndef JF_DUMP_CUH
#define JF_DUMP_CUH
#include "jf_kernels.cuh"

namespace jfk {

constexpr uint32_t DUMP_TP  = 8192;            // original positions per tile
constexpr uint32_t DUMP_NTH = 256;
constexpr uint32_t DUMP_MAXC = DUMP_TP + 8192; // candidates of a tile at most: TP + margin slots (margin <= tri(126) = 8001)

struct DumpArgs {
  TableDev T;
  const uint64_t* inv_lut;     // byte tables of the inverse matrix
  uint32_t nbytes;             // ceil(2k/8)
  uint32_t ocl;                // out_counter_len
  uint64_t seg_lo, seg_hi;     // local original positions of this segment
  uint64_t slots_end;          // local slots that exist (local_size + margin)
  uint64_t margin;             // tri(max_reprobe)
  uint64_t lower, upper;       // count filter
  uint32_t n_tiles;
  uint32_t* tile_cnt;          // [n_tiles + 1]: counts, then exclusive offsets; [n_tiles] = total
  uint8_t* out;                // record bytes of the segment
  uint64_t out_cap;            // records
};

template<int SB>
__global__ void __launch_bounds__(DUMP_NTH) dump_count_kernel(const DumpArgs a) {
  const TableDev& T = a.T;
  const bool any_ovf = T.stats[STAT_OVERFLOWED] != 0;
  __shared__ uint32_t wsum[DUMP_NTH / 32];
  for(uint32_t tile = blockIdx.x; tile < a.n_tiles; tile += gridDim.x) {
    const uint64_t lo = a.seg_lo + (uint64_t)tile * DUMP_TP;
    const uint64_t hi = min(lo + DUMP_TP, a.seg_hi);
    const uint64_t s_end = min(hi + a.margin, a.slots_end);
    uint32_t n = 0;
    for(uint64_t s = lo + threadIdx.x; s < s_end; s += DUMP_NTH) {
      u128 high; uint32_t rp; uint64_t cnt;
      if(!slot_decode<SB>(T, s, high, rp, cnt)) continue;
      const uint64_t opos = s - (rp ? tri(rp) : 0);
      if(opos < lo || opos >= hi) continue;
      if(any_ovf) cnt = slot_full_count<SB>(T, s, cnt);
      if(cnt >= a.lower && cnt <= a.upper) ++n;
    }
#pragma unroll
    for(int o = 16; o; o >>= 1) n += __shfl_xor_sync(0xffffffffu, n, o);
    if((threadIdx.x & 31) == 0) wsum[threadIdx.x >> 5] = n;
    __syncthreads();
    if(threadIdx.x == 0) { uint32_t t = 0; for(uint32_t w = 0; w < DUMP_NTH / 32; ++w) t += wsum[w]; a.tile_cnt[tile] = t; }
    __syncthreads();
  }
}

__global__ void __launch_bounds__(1024) dump_scan_kernel(uint32_t* __restrict__ cnt, uint32_t n) {
  __shared__ uint32_t part[1024];
  const uint32_t per = (n + 1023) / 1024;
  const uint32_t b = threadIdx.x * per, e = min(b + per, n);
  uint32_t s = 0;
  for(uint32_t i = b; i < e; ++i) s += cnt[i];
  part[threadIdx.x] = s;
  __syncthreads();
  for(uint32_t d = 1; d < 1024; d <<= 1) {
    const uint32_t v = threadIdx.x >= d ? part[threadIdx.x - d] : 0;
    __syncthreads();
    part[threadIdx.x] += v;
    __syncthreads();
  }
  uint32_t run = part[threadIdx.x] - s;
  for(uint32_t i = b; i < e; ++i) { const uint32_t c = cnt[i]; cnt[i] = run; run += c; }
  if(threadIdx.x == 1023) cnt[n] = part[1023];
}

template<int KW, int SB>
__global__ void __launch_bounds__(DUMP_NTH) dump_emit_kernel(const DumpArgs a) {
  extern __shared__ __align__(16) uint8_t smem_raw[];
  uint64_t* lut = reinterpret_cast<uint64_t*>(smem_raw);
  uint32_t* cur = reinterpret_cast<uint32_t*>(lut + a.nbytes * 256);     // [TP + 1] counts -> cursors
  uint16_t* list = reinterpret_cast<uint16_t*>(cur + DUMP_TP + 1);       // [DUMP_MAXC] slot offsets from `lo`, grouped by position
  uint8_t* stage = reinterpret_cast<uint8_t*>(list + DUMP_MAXC);         // DUMP_NTH records
  __shared__ uint32_t wtot[DUMP_NTH / 32];
  const TableDev& T = a.T;
  const bool any_ovf = T.stats[STAT_OVERFLOWED] != 0;
  const uint32_t rec = a.nbytes + a.ocl;
  const uint64_t maxv = a.ocl >= 8 ? ~0ull : ((1ull << (8 * a.ocl)) - 1ull);
  for(uint32_t i = threadIdx.x; i < a.nbytes * 256u; i += DUMP_NTH) lut[i] = a.inv_lut[i];

  for(uint32_t tile = blockIdx.x; tile < a.n_tiles; tile += gridDim.x) {
    const uint32_t n_tile = a.tile_cnt[tile + 1] - a.tile_cnt[tile];
    if(n_tile == 0) continue;                                   // (uniform over the CTA)
    const uint64_t lo = a.seg_lo + (uint64_t)tile * DUMP_TP;
    const uint64_t hi = min(lo + DUMP_TP, a.seg_hi);
    const uint64_t s_end = min(hi + a.margin, a.slots_end);
    __syncthreads();
    for(uint32_t i = threadIdx.x; i <= DUMP_TP; i += DUMP_NTH) cur[i] = 0;
    __syncthreads();
    // records per original position
    for(uint64_t s = lo + threadIdx.x; s < s_end; s += DUMP_NTH) {
      u128 high; uint32_t rp; uint64_t cnt;
      if(!slot_decode<SB>(T, s, high, rp, cnt)) continue;
      const uint64_t opos = s - (rp ? tri(rp) : 0);
      if(opos < lo || opos >= hi) continue;
      if(any_ovf) cnt = slot_full_count<SB>(T, s, cnt);
      if(cnt >= a.lower && cnt <= a.upper) atomicAdd(&cur[opos - lo], 1u);
    }
    __syncthreads();
    // exclusive scan of cur[0 .. TP): every thread owns TP / NTH consecutive positions
    {
      constexpr uint32_t PER = DUMP_TP / DUMP_NTH;
      const uint32_t b = threadIdx.x * PER;
      uint32_t s = 0;
#pragma unroll 4
      for(uint32_t i = 0; i < PER; ++i) s += cur[b + i];
      uint32_t incl = s;
#pragma unroll
      for(int o = 1; o < 32; o <<= 1) { const uint32_t v = __shfl_up_sync(0xffffffffu, incl, o); if((threadIdx.x & 31) >= (uint32_t)o) incl += v; }
      if((threadIdx.x & 31) == 31) wtot[threadIdx.x >> 5] = incl;
      __syncthreads();
      uint32_t woff = 0;
      for(uint32_t w = 0; w < (threadIdx.x >> 5); ++w) woff += wtot[w];
      uint32_t run = woff + incl - s;
      for(uint32_t i = 0; i < PER; ++i) { const uint32_t c = cur[b + i]; cur[b + i] = run; run += c; }
    }
    __syncthreads();
    // place the slots: after this pass cur[p] = END of bucket p (its start is the end of bucket p-1)
    for(uint64_t s = lo + threadIdx.x; s < s_end; s += DUMP_NTH) {
      u128 high; uint32_t rp; uint64_t cnt;
      if(!slot_decode<SB>(T, s, high, rp, cnt)) continue;
      const uint64_t opos = s - (rp ? tri(rp) : 0);
      if(opos < lo || opos >= hi) continue;
      if(any_ovf) cnt = slot_full_count<SB>(T, s, cnt);
      if(cnt >= a.lower && cnt <= a.upper) list[atomicAdd(&cur[opos - lo], 1u)] = (uint16_t)(s - lo);
    }
    __syncthreads();
    // order each bucket by the explicit key bits (two keys with one position differ there; heap_item::operator>,
    // mer_heap.hpp:26-30, compares position first, then the key)
    for(uint32_t p = threadIdx.x; p < (uint32_t)(hi - lo); p += DUMP_NTH) {
      const uint32_t b = p ? cur[p - 1] : 0u, e = cur[p];
      for(uint32_t i = b + 1; i < e; ++i) {
        const uint16_t x = list[i];
        if constexpr(SB == SB_WIDE) {            // four-word keys: compared from the most significant word down
          const unsigned long long* sx = wide_slot(T, lo + x);
          uint32_t j = i;
          while(j > b) {
            const unsigned long long* sy = wide_slot(T, lo + list[j - 1]);
            int q = 3;
            while(q > 0 && sy[1 + q] == sx[1 + q]) --q;
            if(sy[1 + q] <= sx[1 + q]) break;
            list[j] = list[j - 1];
            --j;
          }
          list[j] = x;
          continue;
        }
        u128 hx; uint32_t rp; uint64_t c;
        slot_decode<SB>(T, lo + x, hx, rp, c);
        uint32_t j = i;
        while(j > b) {
          u128 hy;
          slot_decode<SB>(T, lo + list[j - 1], hy, rp, c);
          if(hy.hi < hx.hi || (hy.hi == hx.hi && hy.lo <= hx.lo)) break;
          list[j] = list[j - 1];
          --j;
        }
        list[j] = x;
      }
    }
    __syncthreads();
    // emit: DUMP_NTH records per round through the staging buffer
    uint8_t* out = a.out + (uint64_t)a.tile_cnt[tile] * rec;
    for(uint32_t r0 = 0; r0 < n_tile; r0 += DUMP_NTH) {
      const uint32_t i = r0 + threadIdx.x;
      if(i < n_tile) {
        const uint64_t s = lo + list[i];
        u128 high; uint32_t rp; uint64_t cnt;
        slot_decode<SB>(T, s, high, rp, cnt);
        if(any_ovf) cnt = slot_full_count<SB>(T, s, cnt);
        const uint64_t opos = s - (rp ? tri(rp) : 0);
        uint64_t key[KW];
        if constexpr(SB == SB_WIDE) {
#pragma unroll
          for(int q = 0; q < KW; ++q) key[q] = wide_slot(T, s)[1 + q];
        } else key_from_position<KW>(lut, a.nbytes, T.lsize, high, global_pos(T, opos), key);
        uint8_t* d = stage + threadIdx.x * rec;
        for(uint32_t b = 0; b < a.nbytes; ++b) d[b] = (uint8_t)(key[b >> 3] >> ((b & 7) * 8));
        if(cnt > maxv) cnt = maxv;
        for(uint32_t b = 0; b < a.ocl; ++b) d[a.nbytes + b] = (uint8_t)(cnt >> (8 * b));
      }
      __syncthreads();
      const uint32_t nb = min(DUMP_NTH, n_tile - r0) * rec;
      uint8_t* o = out + (uint64_t)r0 * rec;
      for(uint32_t j = threadIdx.x; j < nb; j += DUMP_NTH) o[j] = stage[j];
      __syncthreads();
    }
  }
}

}  // namespace jfk
#endif
