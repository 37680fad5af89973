// jf_shard.cuh -- sharded counting (one engine per GPU, the table split by the top bits of the hash position): the receive side.
//
// Send side: K1 (jf_extract.cuh, FAST form) writes 4-byte records for the regions of the GLOBAL table into a send pool whose
// chunk arenas belong to the owning shards, so a shard's chunks and their directory entries are contiguous and go over
// NVLink as they are (NCCL all-to-all of 8 KB chunks; 4 bytes per k-mer instead of an 8-byte key, no hashing on the
// receiver).  A global region is 1/RING_P of the global table, i.e. `split` regions of the receiver's own partition.
//
// restage_kernel, here: the received chunks -> records of the receiver's own regions, appended to its record pool through the
// same shared-memory rings K1 uses (32-byte stores); K2 then drains that pool exactly as on one GPU.
#ifndef JF_SHARD_CUH
#define JF_SHARD_CUH
#include "jf_extract.cuh"

namespace jfk {

struct RestageArgs {
  TableDev T;
  const uint8_t* recv_pool;      // n_src segments of seg_chunks chunks
  const uint2* recv_dir;         // { global region, records } per received chunk, same indexing
  uint32_t n_src, seg_chunks;
  uint32_t count[8];             // chunks received from every source
  uint32_t first_region;         // first global region this shard owns
  uint32_t split_lg;             // log2(own regions per global region)
  uint32_t sbits;                // log2(slots of a global region)
  const uint8_t* self_pool;      // when not NULL: this shard's own chunks are read where K1 left them (its arena of the send
  const uint2* self_dir;         // bank) instead of travelling through the receive pool; self_src = this shard's rank
  uint32_t self_src, pad0;
  const uint64_t* inv_lut;       // (failure path: the key of a record that found no slot)
  uint32_t nbytes;
};

template<int KW>
__global__ void __launch_bounds__(1024, 1) restage_kernel(const RestageArgs ra, const PartDev pd) {
  constexpr int NTH = 1024;
  extern __shared__ __align__(16) uint8_t rs_smem[];
  uint32_t* st_cnt = reinterpret_cast<uint32_t*>(rs_smem);      // low 16 bits: records handed out, high 16: records written
  uint32_t* st_chunk = st_cnt + RING_P;
  uint32_t* ring = st_chunk + RING_P;
  const uint32_t tid = threadIdx.x;
  const TableDev& T = ra.T;
  const uint32_t hb = T.fbits - T.rbits;
  const uint32_t hmask = hb ? ((1u << hb) - 1u) : 0u;
  const uint32_t fine_bits = pd.region_bits;                    // slots of an own region
  const uint32_t fine_mask = (1u << fine_bits) - 1u;
  uint32_t* my_chunk = pd.cta_chunk + (size_t)blockIdx.x * pd.P;
  uint32_t* my_fill  = pd.cta_fill + (size_t)blockIdx.x * pd.P;
  for(uint32_t p = tid; p < pd.P; p += NTH) {
    uint32_t c = my_chunk[p], f = my_fill[p];
    if(c == NO_CHUNK) c = fresh_chunk(pd, blockIdx.x, T.stats, f);
    st_chunk[p] = c; st_cnt[p] = f | (f << 16);
  }
  __syncthreads();
  const uint32_t rlen = pd.ring_len;
  auto flush_rings = [&](const bool finish) {
    for(uint32_t p = tid; p < pd.P; p += NTH) {
      const uint32_t v = st_cnt[p];
      uint32_t cnt = v & 0xFFFFu, fl = v >> 16;
      const uint32_t lim = min(fl + rlen, pd.chunk_recs);
      if(cnt > lim) cnt = lim;                    // the slots beyond were inserted directly: hand them out again
      const uint32_t c = st_chunk[p];
      if(c == NO_CHUNK) continue;
      uint32_t* dst = reinterpret_cast<uint32_t*>(pd.pool + (size_t)c * CHUNK_BYTES);
      const uint32_t* rg = ring + p * rlen;
      while((fl & 7u) && fl < cnt) { dst[fl] = rg[fl & (rlen - 1)]; ++fl; }
      while(cnt - fl >= 8u) {
        const uint4 x0 = *reinterpret_cast<const uint4*>(rg + (fl & (rlen - 1))), x1 = *reinterpret_cast<const uint4*>(rg + (fl & (rlen - 1)) + 4);
        *reinterpret_cast<uint4*>(dst + fl) = x0; *reinterpret_cast<uint4*>(dst + fl + 4) = x1;
        fl += 8;
      }
      const bool close = cnt + min(rlen, pd.margin) > pd.chunk_recs;
      if(close || finish) for(; fl < cnt; ++fl) dst[fl] = rg[fl & (rlen - 1)];
      if(close) {
        pd.dir[c] = make_uint2(p, cnt);
        const uint32_t nc = alloc_chunk(pd, blockIdx.x);
        st_chunk[p] = nc;
        if(nc == NO_CHUNK) { atomicAdd(&T.stats[STAT_POOL_FULL], 1ull); cnt = fl = pd.chunk_recs; }
        else cnt = fl = 0;
      }
      st_cnt[p] = cnt | (fl << 16);
    }
  };
  // The received chunks, flattened source after source, in batches of NTH per CTA: every THREAD owns one chunk of the batch and a trip
  // of the loop takes the same 16-byte piece (4 records) of all of them.  A chunk holds records of ONE global region -- `split`
  // own regions --, so walking chunk after chunk would pour thousands of records into a handful of rings per trip; across
  // 1024 chunks a trip's 4096 records spread over all the own regions the way K1's do.
  uint32_t total = 0;
  for(uint32_t s = 0; s < ra.n_src; ++s) total += ra.count[s];
  LocalStats ls = { 0, 0, 0, 0, 0 };
  // (chunk j of the list belongs to CTA j mod grid: every CTA gets the same number of chunks to within one, and the
  // chunks of a batch lie far apart in the list)
  for(uint32_t base = 0; base * gridDim.x + blockIdx.x < total; base += NTH) {      // (uniform over the CTA)
    const uint32_t ci = (base + tid) * gridDim.x + blockIdx.x;
    uint32_t n = 0, own = 0;
    const uint4* src = nullptr;
    if(ci < total) {
      uint32_t s = 0, rel = ci;
      while(rel >= ra.count[s]) { rel -= ra.count[s]; ++s; }
      const bool from_self = ra.self_pool != nullptr && s == ra.self_src;
      const size_t at = from_self ? (size_t)rel : (size_t)s * ra.seg_chunks + rel;
      const uint2 d = __ldg(from_self ? &ra.self_dir[at] : &ra.recv_dir[at]);
      n = d.y;
      own = (d.x - ra.first_region) << ra.split_lg;              // first own region of that global region
      src = reinterpret_cast<const uint4*>((from_self ? ra.self_pool : ra.recv_pool) + at * CHUNK_BYTES);
    }
    // (chunks are full but for the last of every (CTA, region) pair of the sender: most trips are needed by most threads)
    uint32_t n_max = n;
#pragma unroll
    for(int o = 16; o; o >>= 1) n_max = max(n_max, __shfl_xor_sync(0xffffffffu, n_max, o));
    __shared__ uint32_t s_nmax;
    if(tid == 0) s_nmax = 0;
    __syncthreads();
    if((tid & 31) == 0) atomicMax(&s_nmax, n_max);
    __syncthreads();
    // two pieces (8 records) per thread and trip: half the ring passes; the pieces of the next trip are already on their way
    const uint32_t trips = (s_nmax + 7) / 8;
    uint4 nx0 = make_uint4(0, 0, 0, 0), nx1 = make_uint4(0, 0, 0, 0);
    if(0 < n) nx0 = __ldg(src);
    if(4 < n) nx1 = __ldg(src + 1);
    for(uint32_t trip = 0; trip < trips; ++trip) {
      const uint4 v0 = nx0, v1 = nx1;
      const uint32_t r0 = trip * 8;
      if(r0 + 8 < n) nx0 = __ldg(src + 2 * trip + 2);
      if(r0 + 12 < n) nx1 = __ldg(src + 2 * trip + 3);
      if(r0 < n) {
        const uint32_t rec[8] = { v0.x, v0.y, v0.z, v0.w, v1.x, v1.y, v1.z, v1.w };
#pragma unroll
        for(uint32_t q = 0; q < 8; ++q) {
          if(r0 + q >= n) break;
          const uint32_t pos = rec[q] >> hb, high = rec[q] & hmask;            // position inside the global region
          const uint32_t p = own + (pos >> fine_bits);
          const uint32_t r2 = ((pos & fine_mask) << hb) | high;
          const uint32_t w = atomicAdd(&st_cnt[p], 1u);
          const uint32_t slot = w & 0xFFFFu, fl = w >> 16;
          if(slot - fl < rlen && slot < pd.chunk_recs) ring[p * rlen + (slot & (rlen - 1))] = r2;
          else {
            // ring or chunk full (skewed input): straight into the table -- no window kernel runs beside this one
            u128 hh; hh.lo = high; hh.hi = 0;
            const uint64_t slot_base = ((uint64_t)p << fine_bits) + (pos & fine_mask);
            if(table_add_hp<32>(T, slot_base, hh, 1, ls)) ls.inserted++;
            else k2_fail<KW>(T.shard_index, T.local_lsize, T.lsize, T.stats, T.fail_keys, T.fail_counts, T.fail_cap, slot_base, high, ra.inv_lut, ra.nbytes);
          }
        }
      }
      __syncthreads();
      flush_rings(false);
      __syncthreads();
    }
  }
  flush_rings(true);
  __syncthreads();
  for(uint32_t p = tid; p < pd.P; p += NTH) { my_chunk[p] = st_chunk[p]; my_fill[p] = min(st_cnt[p] & 0xFFFFu, pd.chunk_recs); }
  flush_stats(T.stats, ls.inserted, ls.distinct, ls.reprobes);
}

}  // namespace jfk
#endif
