// jf_window.cuh -- K2, the shared-memory window insert (the default form of K2 for 32-bit slots and 4-byte records).
//
// The L2 form of K2 (insert_chunks32_kernel) performs ~2 L2 operations per k-mer (first-probe CAS, reprobes,
// look-ahead loads).  Here the probing happens in shared memory:
//   win_scatter<true> / win_scan / win_scatter<false>  split the 4-byte records of a group of regions by WINDOW
//        (2^WIN_LG slots = 64 KB of 32-bit slots) with a shared-memory staged tile sort, so that each
//        window's records are contiguous (8 B of traffic per record).  The bucket pass puts every window's records
//        into a bucket of fixed capacity (wd.cap), so it needs no count beforehand; its atomics on the window
//        cursors leave the exact count of every window behind.  A window that overflows its bucket flags the group,
//        and only then does the exact pass place the group's records again, at offsets scanned from those counts;
//   win_insert2  persistent, one CTA per SM, two stages: while the CTA applies the records of one window with
//        shared-memory CAS/add along the reference's probe sequence pos + i(i+1)/2, the TMA engine brings in the
//        next window and its records (cp.async.bulk + mbarrier) and writes the previous window back
//        (cp.async.bulk shared -> global): 8 B of table traffic per slot + 4 B per record, no global-memory
//        latency inside the probing loop.  A probe that would leave the window is DEFERRED (position + key
//        bits appended to a list); a counter carry goes to the side overflow table exactly as in the L2 kernels;
//   win_deferred  the deferred records, with the ordinary global probe sequence, after win_insert
//        of the same group has completed (stream order), so no slot is ever touched by a window CTA
//        and by the global path at the same time.
// The first drain after the table was cleared is WRITE-ONLY (WinDev::lazy_win): the table's slots were not zeroed in memory
// (jf_engine.cu, table_zero), so win_insert2 zeroes each stage in shared memory instead of loading the window, and
// win_zero writes the windows that receive no record.  The table then crosses HBM once per drain instead of three times
// (memset, load, store).  The few windows K1 put in memory for a direct insertion (lazy_win_materialize) are loaded and
// kept as usual.  A deferred probe of a group's last window may reach into the next group's first window, which
// that group's win_insert2 writes without reading: the engine applies a group's deferred records after the NEXT group's
// win_insert2 (two deferred lists).
// Slots only ever fill up, so a key that left its window because every slot of its sequence inside
// the window belongs to other keys finds the same situation on every later visit: all its
// occurrences are deferred, and it cannot end up in two slots.
#pragma once

namespace jfk {

constexpr uint32_t WIN_MAX_G = 64;                 // regions per group
constexpr uint32_t WIN_MAX_WPR = 2048;             // windows per region (region_bits - WIN_LG <= 11)

struct WinDev {
  uint32_t g0, G, wpr_lg, n_tiles;                 // n_tiles: win_scatter's tiles of the group
  uint32_t cap;                                    // records per window bucket (a multiple of 4: buckets start on 16-byte boundaries)
  const uint32_t* lazy_win;                        // write-only drain: the table's window states (only WIN_IN_MEMORY windows are loaded); else null
  uint32_t stile_first[WIN_MAX_G + 1];             // prefix sum of win_scatter's tiles (WIN_ST_UNITS chunks) per region of the group
  uint32_t unit_first[WIN_MAX_G + 1];              // first unit (index into `order`) of each region; [G] = end
  uint32_t* overflow;                              // the group's flag: some window holds more than `cap` records
  uint32_t* wstart;                                // [(G << wpr_lg) + 1] offsets into wrec after win_scan
  uint32_t* wcursor;                               // [G << wpr_lg] counts (bucket pass), then write cursors (exact pass)
  uint32_t* wcnt;                                  // [G << wpr_lg] records per window (win_scan); runs start on 16-byte boundaries
  uint32_t* wrec; uint64_t wrec_cap;               // records grouped by (region, window)
  uint64_t* def_pos; uint32_t* def_high; unsigned long long* def_n; uint64_t def_cap;
};

// first slot of window `task` (= region of the group << wpr_lg | window of the region)
__device__ __forceinline__ uint64_t win_slot_base(const WinDev& wd, uint32_t region_bits, uint32_t task) {
  return ((uint64_t)(wd.g0 + (task >> wd.wpr_lg)) << region_bits) + ((uint64_t)(task & ((1u << wd.wpr_lg) - 1)) << WIN_LG);
}

// ---- run starts of the windows (one CTA) --------------------------------------------------------
// After the bucket pass wcursor holds every window's count.  Group not flagged: window i's run is bucket i.  Flagged: the exact
// layout, an exclusive scan of the counts, which also sets wcursor to the run starts for the exact pass.
__global__ void __launch_bounds__(1024) win_scan_kernel(WinDev wd, unsigned long long* __restrict__ stats) {
  __shared__ uint32_t part[1024];
  const uint32_t n = wd.G << wd.wpr_lg;
  if(*wd.overflow == 0) {
    for(uint32_t i = threadIdx.x; i < n; i += 1024) { wd.wstart[i] = i * wd.cap; wd.wcnt[i] = wd.wcursor[i]; }
    if(threadIdx.x == 0) wd.wstart[n] = n * wd.cap;
    return;
  }
  const uint32_t per = (n + 1023) / 1024;
  const uint32_t b = threadIdx.x * per, e = min(b + per, n);
  uint32_t s = 0;
  for(uint32_t i = b; i < e; ++i) s += (wd.wcursor[i] + 3u) & ~3u;
  part[threadIdx.x] = s;
  __syncthreads();
  for(uint32_t d = 1; d < 1024; d <<= 1) {
    const uint32_t v = threadIdx.x >= d ? part[threadIdx.x - d] : 0;
    __syncthreads();
    part[threadIdx.x] += v;
    __syncthreads();
  }
  // every window's run starts on a 16-byte boundary (the TMA engine copies it): counts are rounded up to 4 records
  uint32_t run = part[threadIdx.x] - s;            // exclusive prefix of this thread's segment
  for(uint32_t i = b; i < e; ++i) {
    const uint32_t c = wd.wcursor[i];
    wd.wstart[i] = run; wd.wcursor[i] = run; wd.wcnt[i] = c;
    run += (c + 3u) & ~3u;
  }
  if(threadIdx.x == 1023) {
    wd.wstart[n] = part[1023];
    if(part[1023] > wd.wrec_cap) atomicAdd(&stats[STAT_POOL_FULL], 1ull);   // the host sizes groups so that this cannot happen
  }
}

// ---- tile sort by window, runs written to the group buffer ----------------------------------------
// A tile = WIN_ST_UNITS chunks of one region (24 K records).  A persistent grid, one CTA of WIN_ST_NTH threads per SM, strides
// over the group's tiles.  WIN_ST_NBUF tiles sit in shared memory at a time: while the CTA sorts and stores one, the TMA
// engine brings in the next (cp.async.bulk + mbarrier), so every record is read from HBM once.  Each thread holds its
// records in registers, and with each record its rank inside its window, which the histogram's shared-memory atomicAdd
// returns; after the scan the records go back into the same buffer, sorted by window, and the runs (one per window, ~48
// records at configs[1]) go to their places in the group buffer with coalesced stores.  Three block barriers per tile:
// histogram complete (the previous tile's buffer is free: the next load is issued), warp totals of the scan, placement
// complete.  The global atomicAdd that gives a run its place is issued before the placement and used after it.
// BUCKETS (the bucket pass): the run of window gw goes to bucket gw after what earlier tiles put there; a run that would
// overflow the bucket is not stored and flags the group.  Either way its length is added to wcursor[gw], so the pass leaves
// every window's exact count behind.  Once a CTA sees the flag it sorts and stores nothing more, but still counts: the
// group is placed again by the exact pass (!BUCKETS), which returns at once when the flag is clear and otherwise stores
// every run at the start win_scan gave it.
constexpr uint32_t WIN_ST_UNITS = 12;              // chunks per tile: the longest runs two tile buffers leave room for
constexpr uint32_t WIN_ST_NBUF = 2;                // tiles in shared memory
constexpr uint32_t WIN_ST_NTH = 1024;

// dynamic shared memory of win_scatter_kernel: the tile buffers, then cnt, lbase and gbase (one word per window of a region)
__host__ __device__ constexpr size_t win_scatter_smem(uint32_t units, uint32_t nbuf, uint32_t wpr) {
  return (size_t)nbuf * units * CHUNK_BYTES + (size_t)3 * wpr * 4;
}
static_assert(win_scatter_smem(WIN_ST_UNITS, WIN_ST_NBUF, WIN_MAX_WPR) + 1024 <= 227 * 1024, "one CTA per SM");

// (a persistent CTA of NTH threads; UNITS, NBUF and NTH are parameters so that scripts/micro/win_scatter.cu can compare tile shapes)
template<bool BUCKETS, uint32_t UNITS, uint32_t NBUF, uint32_t NTH>
__device__ __forceinline__ void win_scatter_tiles(const PartDev& pd, const WinDev& wd, const uint32_t* __restrict__ order, uint32_t hb) {
  constexpr uint32_t CR = CHUNK_BYTES / 4;         // records per chunk (the window form takes 4-byte records only)
  constexpr uint32_t V = UNITS * (CHUNK_BYTES / 16) / NTH;     // 16-byte pieces of a tile per thread
  constexpr uint32_t PER_MAX = NTH >= WIN_MAX_WPR ? 1 : NTH * 2 >= WIN_MAX_WPR ? 2 : 4;     // windows per thread in the scan
  static_assert(UNITS * (CHUNK_BYTES / 16) % NTH == 0 && NTH % 32 == 0 && NTH * PER_MAX >= WIN_MAX_WPR && NBUF >= 2 && UNITS <= 32, "tile shape");
  static_assert(UNITS * CR <= 65536, "ranks are packed two to a word");
  extern __shared__ __align__(128) uint32_t wsm[];
  __shared__ __align__(8) uint64_t full[NBUF];
  __shared__ uint32_t s_n[NBUF][UNITS];            // records of each chunk of the tile in each buffer
  __shared__ uint32_t warp_tot[NTH / 32];
  __shared__ uint32_t s_skip;
  if(!BUCKETS && *wd.overflow == 0) return;
  const uint32_t wpr = 1u << wd.wpr_lg, wmask = wpr - 1;
  uint32_t per_lg = 0;                             // (NTH << per_lg >= wpr)
  while((NTH << per_lg) < wpr) ++per_lg;
  const uint32_t per = 1u << per_lg;
  uint32_t* const cnt = wsm + NBUF * UNITS * CR;
  uint32_t* const lbase = cnt + wpr;               // warp-local exclusive prefix of the window counts
  uint32_t* const gbase = lbase + wpr;             // output position = this + index in the sorted tile
  const uint32_t tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
  const uint32_t n_mine = blockIdx.x < wd.n_tiles ? (wd.n_tiles - 1 - blockIdx.x) / gridDim.x + 1 : 0;
  auto region_of = [&](uint32_t tile) { uint32_t r = 0; while(r + 1 < wd.G && wd.stile_first[r + 1] <= tile) ++r; return r; };
  // warp 0, lane j < UNITS: chunk j of this CTA's k-th tile (NO_CHUNK past the tile's end), and its records
  auto chunk_of = [&](uint32_t k) -> uint32_t {
    if(k >= n_mine || lane >= UNITS) return NO_CHUNK;
    const uint32_t tile = blockIdx.x + k * gridDim.x, r = region_of(tile);
    const uint32_t u = wd.unit_first[r] + (tile - wd.stile_first[r]) * UNITS + lane;
    return u < wd.unit_first[r + 1] ? __ldg(order + u) : NO_CHUNK;
  };
  auto recs_of = [&](uint32_t c) -> uint32_t { return c != NO_CHUNK ? min(__ldg(&pd.dir[c].y), CR) : 0u; };
  // warp 0: the TMA engine brings this CTA's k-th tile into buffer k % NBUF
  auto issue = [&](uint32_t k, uint32_t c, uint32_t n) {
    const uint32_t b = k % NBUF, bytes = ((n + 3u) & ~3u) * 4u;
    uint32_t sum = bytes;
#pragma unroll
    for(int o = 16; o; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    if(lane < UNITS) s_n[b][lane] = n;
    __syncwarp();
    if(lane == 0) { fence_proxy_async(); mbar_expect_tx(&full[b], sum); }   // (s_n is released by this arrival)
    __syncwarp();
    if(bytes) tma_load_1d(wsm + (b * UNITS + lane) * CR, pd.pool + (size_t)c * CHUNK_BYTES, bytes, &full[b]);
  };

  if(tid == 0) {
    for(uint32_t b = 0; b < NBUF; ++b) mbar_init(&full[b], 1);
    fence_proxy_async();
    s_skip = 0;
  }
  for(uint32_t i = tid; i < wpr; i += NTH) cnt[i] = 0;
  __syncthreads();
  uint32_t pc = NO_CHUNK, pn = 0;                  // warp 0: the next tile to issue (k + NBUF - 1 at tile k)
  if(warp == 0) {
    for(uint32_t k = 0; k + 1 < NBUF && k < n_mine; ++k) { const uint32_t c = chunk_of(k); issue(k, c, recs_of(c)); }
    pc = chunk_of(NBUF - 1); pn = recs_of(pc);
  }
  bool skip = false;                               // (BUCKETS) the group's flag was seen: count only

  for(uint32_t k = 0; k < n_mine; ++k) {
    const uint32_t b = k % NBUF;
    uint32_t* const buf = wsm + b * UNITS * CR;
    mbar_wait(&full[b], (k / NBUF) & 1u);
    // histogram; the rank a record gets there is its place in its window's run
    uint32_t rec[4 * V], rank[2 * V];
#pragma unroll
    for(uint32_t v = 0; v < V; ++v) {
      const uint32_t x = tid + v * NTH, j = x / (CR / 4), q0 = (x % (CR / 4)) * 4, n = s_n[b][j];
      const uint4 r4 = reinterpret_cast<const uint4*>(buf)[x];
      rec[4 * v] = r4.x; rec[4 * v + 1] = r4.y; rec[4 * v + 2] = r4.z; rec[4 * v + 3] = r4.w;
      rank[2 * v] = rank[2 * v + 1] = 0;
#pragma unroll
      for(uint32_t q = 0; q < 4; ++q)
        if(q0 + q < n) rank[2 * v + q / 2] |= atomicAdd(&cnt[((rec[4 * v + q] >> hb) >> WIN_LG) & wmask], 1u) << (16 * (q & 1));
    }
    __syncthreads();                               // (1) histogram complete, the previous tile's buffer stored
    if(warp == 0 && k + NBUF - 1 < n_mine) { issue(k + NBUF - 1, pc, pn); pc = chunk_of(k + NBUF); }
    // exclusive scan of cnt: thread tid owns windows [tid * per, tid * per + per)
    const uint32_t i0 = tid << per_lg;
    uint32_t c[PER_MAX], s = 0;
#pragma unroll
    for(uint32_t p = 0; p < PER_MAX; ++p) { c[p] = p < per && i0 < wpr ? cnt[i0 + p] : 0u; s += c[p]; }
    uint32_t incl = s;
#pragma unroll
    for(int o = 1; o < 32; o <<= 1) { const uint32_t v = __shfl_up_sync(0xffffffffu, incl, o); if(lane >= (uint32_t)o) incl += v; }
    if(lane == 31) warp_tot[warp] = incl;
    if(i0 < wpr) {
      uint32_t x = incl - s;
#pragma unroll
      for(uint32_t p = 0; p < PER_MAX; ++p) if(p < per) { lbase[i0 + p] = x; x += c[p]; cnt[i0 + p] = 0; }
    }
    __syncthreads();                               // (2) warp totals
    const uint32_t wt = lane < NTH / 32 ? warp_tot[lane] : 0u;
    uint32_t winc = wt;
#pragma unroll
    for(int o = 1; o < 32; o <<= 1) { const uint32_t v = __shfl_up_sync(0xffffffffu, winc, o); if(lane >= (uint32_t)o) winc += v; }
    const uint32_t wexcl = winc - wt, total = __shfl_sync(0xffffffffu, winc, 31);
    // the runs' places: in the bucket pass the atomics are in flight while the records are placed
    const uint32_t run0 = __shfl_sync(0xffffffffu, wexcl, warp) + incl - s;
    const uint32_t r = region_of(blockIdx.x + k * gridDim.x);
    uint32_t at[PER_MAX];
    auto claim = [&] {
#pragma unroll
      for(uint32_t p = 0; p < PER_MAX; ++p) at[p] = c[p] ? atomicAdd(&wd.wcursor[(r << wd.wpr_lg) + i0 + p], c[p]) : 0u;
    };
    if(BUCKETS) claim();
    uint32_t flag = 0;
    if(BUCKETS && tid == 0) flag = *(volatile uint32_t*)wd.overflow;
    if(!skip) {
#pragma unroll
      for(uint32_t v = 0; v < V; ++v) {
        const uint32_t x = tid + v * NTH, j = x / (CR / 4), q0 = (x % (CR / 4)) * 4, n = s_n[b][j];
#pragma unroll
        for(uint32_t q = 0; q < 4; ++q) {
          const uint32_t w = ((rec[4 * v + q] >> hb) >> WIN_LG) & wmask;
          const uint32_t off = __shfl_sync(0xffffffffu, wexcl, (w >> per_lg) >> 5);
          if(q0 + q < n) buf[lbase[w] + off + ((rank[2 * v + q / 2] >> (16 * (q & 1))) & 0xFFFFu)] = rec[4 * v + q];
        }
      }
    }
    if(!BUCKETS) claim();                          // (the exact pass, run only for a flagged group: after the placement, which
                                                   // leaves no register for the atomics in flight)
    if(i0 < wpr) {
      uint32_t run = run0;
#pragma unroll
      for(uint32_t p = 0; p < PER_MAX; ++p) if(p < per) {
        uint32_t a = at[p];
        if(BUCKETS && c[p]) {
          const uint32_t gw = (r << wd.wpr_lg) + i0 + p;
          if(a + c[p] <= wd.cap) a += gw * wd.cap;
          else { a = (uint32_t)wd.wrec_cap; *(volatile uint32_t*)wd.overflow = 1u; flag = 1; }   // (every store of the run is past wrec_cap)
        }
        gbase[i0 + p] = a - run;
        run += c[p];
      }
    }
    if(BUCKETS && flag) s_skip = 1;
    fence_proxy_async();                           // the placement's writes, before the TMA engine refills this buffer
    __syncthreads();                               // (3) placement and run starts complete
    if(BUCKETS) skip = s_skip != 0;
    if(!skip) {
      for(uint32_t i = tid; i < total; i += NTH) {
        const uint32_t v = buf[i], w = ((v >> hb) >> WIN_LG) & wmask;
        const uint32_t dst = gbase[w] + i;
        if(dst < wd.wrec_cap) wd.wrec[dst] = v;
      }
    }
    if(warp == 0) pn = recs_of(pc);                // (its latency is hidden behind the next tile's histogram)
  }
}

template<bool BUCKETS>
__global__ void __launch_bounds__(WIN_ST_NTH, 1) win_scatter_kernel(PartDev pd, WinDev wd, const uint32_t* __restrict__ order, uint32_t hb) {
  win_scatter_tiles<BUCKETS, WIN_ST_UNITS, WIN_ST_NBUF, WIN_ST_NTH>(pd, wd, order, hb);
}

// ---- persistent window insert: probe in shared memory, windows and records moved by the TMA engine -------------
// Warp 0 is the PRODUCER: it finds this CTA's next non-empty window, brings the window and its records into one of two
// stages (cp.async.bulk + mbarrier `full`), and, once the consumers have released a stage (mbarrier `empty`), writes the
// window back (cp.async.bulk shared -> global) and refills the stage.  Warps 1..31 are CONSUMERS: they never meet at a
// block-wide barrier -- a warp that runs out of records in one stage moves on to the other one.
constexpr uint32_t WIN2_NTH = 1024;
constexpr uint32_t WIN2_CONS = WIN2_NTH - 32;      // consumer threads
constexpr uint32_t WIN2_RB  = 10240;               // records per batch (a window of iid input holds ~0.6 * WIN_SLOTS)
constexpr uint32_t WIN2_BLK = 256;                 // records a consumer warp claims at a time
constexpr uint32_t WIN2_NONE = 0xFFFFFFFFu;
constexpr size_t   WIN2_SMEM = (size_t)2 * WIN_SLOTS * 4 + (size_t)2 * WIN2_RB * 4;

struct Win2Info { uint32_t task, b, n, pad; };

template<int KW>
__global__ void __launch_bounds__(WIN2_NTH, 1) win_insert2_kernel(TableDev T, PartDev pd, WinDev wd, const uint64_t* __restrict__ inv_lut_g, uint32_t nbytes) {
  extern __shared__ __align__(128) uint8_t w2smem[];
  __shared__ __align__(8) uint64_t full[2];
  __shared__ __align__(8) uint64_t empty[2];
  __shared__ Win2Info info[2];
  __shared__ uint32_t cursor[2];                   // next unclaimed record of the batch in each stage
  uint32_t* const winb0 = reinterpret_cast<uint32_t*>(w2smem);
  uint32_t* const recb0 = winb0 + 2 * WIN_SLOTS;
  uint32_t* tab = (uint32_t*)T.slots;
  const uint32_t n_tasks = wd.G << wd.wpr_lg;
  const uint32_t tid = threadIdx.x, lane = tid & 31u;

  auto slot_base_of = [&](uint32_t task) -> uint64_t { return win_slot_base(wd, pd.region_bits, task); };
  if(tid == 0) {
    mbar_init(&full[0], 1); mbar_init(&full[1], 1);
    mbar_init(&empty[0], WIN2_CONS / 32); mbar_init(&empty[1], WIN2_CONS / 32);     // one arrival per consumer warp
    fence_proxy_async();
  }
  __syncthreads();

  if(tid < 32) {
    // ================================= producer =================================
    // Lane 0 drives the TMA engine and the barriers; every lane follows the same (uniform) control flow, so that in a
    // write-only drain the whole warp can zero a stage in place of loading the window.
    const bool lead = lane == 0;
    uint32_t next_from = blockIdx.x;
    uint32_t ephase[2] = { 0, 0 };
    uint32_t cur_task[2] = { WIN2_NONE, WIN2_NONE }, cur_n[2] = { 0, 0 }, cur_b[2] = { 0, 0 };
    auto load_batch = [&](uint32_t s, uint32_t off, bool with_window) {     // (lead)
      const uint32_t nb = min(WIN2_RB, cur_n[s] - off);
      const uint32_t rbytes = ((nb + 3u) & ~3u) * 4u;
      cursor[s] = 0;
      mbar_expect_tx(&full[s], rbytes + (with_window ? WIN_SLOTS * 4u : 0u));
      if(with_window) tma_load_1d(winb0 + s * WIN_SLOTS, tab + slot_base_of(cur_task[s]), WIN_SLOTS * 4u, &full[s]);
      tma_load_1d(recb0 + s * WIN2_RB, wd.wrec + cur_b[s] + off, rbytes, &full[s]);
    };
    auto next_window = [&](uint32_t s) {             // the next non-empty window of this CTA's stride into stage s
      uint32_t t = next_from, c = 0;
      while(t < n_tasks && (c = wd.wcnt[t]) == 0) t += gridDim.x;
      if(t >= n_tasks) {
        next_from = t; cur_task[s] = WIN2_NONE;
        if(lead) { info[s].task = WIN2_NONE; mbar_arrive(&full[s]); }
        return;
      }
      next_from = t + gridDim.x;
      cur_task[s] = t; cur_n[s] = c; cur_b[s] = wd.wstart[t];
      const bool fill = wd.lazy_win && wd.lazy_win[slot_base_of(t) >> WIN_LG] != WIN_IN_MEMORY;
      if(fill) {
        uint4* const w = reinterpret_cast<uint4*>(winb0 + s * WIN_SLOTS);
        for(uint32_t i = lane; i < WIN_SLOTS / 4; i += 32) w[i] = make_uint4(0, 0, 0, 0);
        fence_proxy_async();                         // these writes, before the TMA engine stores the stage
        __syncwarp();
      }
      if(lead) {
        info[s].task = t; info[s].b = cur_b[s]; info[s].n = c;
        load_batch(s, 0, !fill);
      }
    };
    next_window(0); next_window(1);
    for(uint32_t s = 0; cur_task[s] != WIN2_NONE; s ^= 1u) {
      // the consumers work through the batches of stage s in order
      for(uint32_t off = WIN2_RB; off < cur_n[s]; off += WIN2_RB) {
        mbar_wait(&empty[s], ephase[s]); ephase[s] ^= 1u;
        if(lead) load_batch(s, off, false);
      }
      mbar_wait(&empty[s], ephase[s]); ephase[s] ^= 1u;   // every consumer warp is done with this window
      if(lead) {
        tma_store_1d(tab + slot_base_of(cur_task[s]), winb0 + s * WIN_SLOTS, WIN_SLOTS * 4u);
        tma_commit_group();
        tma_wait_group_read0();                    // the stage may be overwritten
      }
      __syncwarp();
      next_window(s);
    }
    if(lead) tma_wait_group0();                    // every window is back in the table before the kernel ends
    return;
  }

  // ================================= consumers =================================
  const uint32_t fb = T.fbits, rb = T.rbits, hb = fb - rb;
  const uint32_t fmask = (1u << fb) - 1u, one = 1u << fb, cb = 32 - fb;
  const uint32_t hmask = hb ? ((1u << hb) - 1u) : 0u;
  const uint32_t lt_mask = (1u << lane) - 1u;
  uint32_t n_ins = 0, n_new = 0, n_rep = 0;
  uint32_t fphase[2] = { 0, 0 };
  for(uint32_t s = 0; ; s ^= 1u) {
    mbar_wait(&full[s], fphase[s]); fphase[s] ^= 1u;
    const Win2Info inf = info[s];
    if(inf.task == WIN2_NONE) break;               // (the same for every consumer)
    uint32_t* const win = winb0 + s * WIN_SLOTS;
    const uint32_t* const recs = recb0 + s * WIN2_RB;
    const uint64_t slot_base = slot_base_of(inf.task);
    for(uint32_t off = 0; off < inf.n; off += WIN2_RB) {
      const uint32_t nb = min(WIN2_RB, inf.n - off);
      if(off) { mbar_wait(&full[s], fphase[s]); fphase[s] ^= 1u; }
      // Every lane keeps one record in flight and performs ONE probe per trip of the loop; the lanes whose record is settled
      // take the next records of the warp's current block (WIN2_BLK records, claimed with one shared-memory atomic per block;
      // inside a block the indices come from a warp-uniform register counter and a ballot), so a warp stays full until the
      // batch is exhausted whatever the lengths of the probe sequences.
      bool have = false, want = true;
      uint32_t rec = 0, local = 0, kf = 0, at = 0, p = 0;
      uint32_t blk_next = 0, blk_end = 0;          // (warp-uniform)
      bool more = true;                            // the batch may still have unclaimed blocks (warp-uniform)
      for(;;) {
        const uint32_t need = __ballot_sync(0xffffffffu, want);
        if(need && more) {
          if(blk_next >= blk_end) {                // claim the next block
            uint32_t base = 0;
            if(lane == 0) base = atomicAdd(&cursor[s], WIN2_BLK);
            blk_next = __shfl_sync(0xffffffffu, base, 0);
            blk_end = min(blk_next + WIN2_BLK, nb);
            more = blk_next < nb;
          }
          if(want && more) {
            const uint32_t i = blk_next + __popc(need & lt_mask);
            if(i < blk_end) {
              rec = recs[i];
              local = (rec >> hb) & (WIN_SLOTS - 1); kf = ((rec & hmask) << rb) | 1u;
              at = local; p = 0;
              have = true; want = false;
            }                                      // (else: asks again on the next trip, from the next block)
          }
          blk_next = min(blk_next + (uint32_t)__popc(need), blk_end);
        }
        if(!__any_sync(0xffffffffu, have)) { if(!more) break; else continue; }
        if(have) {
          if(at < WIN_SLOTS) {
            const uint32_t o = atomicCAS(&win[at], 0u, kf | one);
            if(o == 0u) { ++n_new; ++n_ins; n_rep += p; want = true; }
            else if((o & fmask) == kf) {
              const uint32_t o2 = atomicAdd(&win[at], one);
              if((((o2 >> fb) + 1) >> cb) != 0) k2_carry(T.ovf_keys, T.ovf_vals, T.ovf_mask, T.stats, slot_base + at);
              ++n_ins; n_rep += p; want = true;
            } else if(p < T.max_reprobe) { ++p; at += p; ++kf; }            // pos + i(i+1)/2, reprobe field + 1
            else {
              k2_fail<KW>(T.shard_index, T.local_lsize, T.lsize, T.stats, T.fail_keys, T.fail_counts, T.fail_cap, slot_base + local, rec & hmask, inv_lut_g, nbytes);
              want = true;
            }
          } else {                                 // leaves the window: the global path takes it after this kernel
            const unsigned long long d = atomicAdd(wd.def_n, 1ull);
            if(d < wd.def_cap) { wd.def_pos[d] = slot_base + local; wd.def_high[d] = rec & hmask; }
            else atomicAdd(&T.stats[STAT_POOL_FULL], 1ull);
            want = true;
          }
          have = !want;
        }
      }
      fence_proxy_async();                         // this thread's writes to the window, before the TMA engine reads it
      __syncwarp();
      if(lane == 0) mbar_arrive(&empty[s]);        // this warp is done with the batch
    }
  }
  flush_stats(T.stats, n_ins, n_new, n_rep);
}

// ---- lazily zeroed table: windows [w_first, w_first + n) that are not in memory yet are written as zeros, except those that
// receive records (wcnt[i] != 0, win_insert2 writes them; wcnt null: none does) -------------------------------------------
__global__ void __launch_bounds__(256) win_zero_kernel(uint32_t* __restrict__ tab, const uint32_t* __restrict__ state, const uint32_t* __restrict__ wcnt,
                                                       uint64_t w_first, uint32_t n) {
  const uint32_t lane = threadIdx.x & 31u;
  const uint32_t n_warps = gridDim.x * (blockDim.x / 32);
  for(uint32_t t = (blockIdx.x * blockDim.x + threadIdx.x) / 32; t < n; t += n_warps) {
    if((wcnt && wcnt[t]) || state[w_first + t] == WIN_IN_MEMORY) continue;
    uint4* const w = reinterpret_cast<uint4*>(tab + ((w_first + t) << WIN_LG));
    for(uint32_t i = lane; i < WIN_SLOTS / 4; i += 32) w[i] = make_uint4(0, 0, 0, 0);
  }
}

// ---- the deferred records: ordinary probe sequence in global memory ---------------------------------
template<int KW>
__global__ void __launch_bounds__(256) win_deferred_kernel(TableDev T, WinDev wd, const uint64_t* __restrict__ inv_lut_g, uint32_t nbytes) {
  const uint32_t one = 1u << T.fbits;
  uint32_t* tab = (uint32_t*)T.slots;
  const unsigned long long n = min(*wd.def_n, (unsigned long long)wd.def_cap);
  uint32_t n_ins = 0, n_new = 0, n_rep = 0;
  for(unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (unsigned long long)gridDim.x * blockDim.x) {
    const uint64_t base = wd.def_pos[i];
    const uint32_t high = wd.def_high[i];
    const uint32_t o = atomicCAS(&tab[base], 0u, ((high << T.rbits) | 1u) | one);
    k2_settle<KW>(T, tab, base, high, o, inv_lut_g, nbytes, n_ins, n_new, n_rep);
  }
  flush_stats(T.stats, n_ins, n_new, n_rep);
}

}  // namespace jfk
