// The bucket pass of K2 (win_scatter_kernel<true>, jf_window.cuh) alone, at the geometry of bench.py's configs[1]: one group
// of 12 regions of 2^23 slots (512 windows of 2^14 slots each), ~2384 chunks of 2048 hashed 4-byte records per region,
// the chunks scattered over the pool as K1's arenas leave them.  Times the kernel over many launches with CUDA events at
// several tile sizes, next to the previous form of the pass (two reads of every chunk, one CTA per tile, copied below as
// `old_scatter_kernel`) and a device-to-device cudaMemcpy of the same bytes.  GB/s counts the algorithmic bytes: every
// record read once and written once (8 B).  Every form's buckets are checked against the host's per-window counts and sums.
//
//   nvcc -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a --expt-relaxed-constexpr -o win_scatter win_scatter.cu
#include <cstdio>
#include <cstdlib>
#include <cstdint>
#include <cmath>
#include <vector>
#include <algorithm>
#include <random>
#include <string>
#include <cstring>
#include "../../jellyfish_b200/csrc/jf_kernels.cuh"
#include "../../jellyfish_b200/csrc/jf_window.cuh"

using namespace jfk;

#define CK(x) do { cudaError_t e_ = (x); if(e_ != cudaSuccess) { fprintf(stderr, "%s:%d %s\n", __FILE__, __LINE__, cudaGetErrorString(e_)); exit(1); } } while(0)

// ---- the previous bucket pass: one CTA per tile of 12 chunks, 2 CTAs per SM, chunks read twice ------------------------
constexpr uint32_t OLD_UNITS = 12;
__global__ void __launch_bounds__(1024, 2) old_scatter_kernel(PartDev pd, WinDev wd, const uint32_t* __restrict__ order, uint32_t hb) {
  extern __shared__ __align__(16) uint32_t osm[];
  const uint32_t wpr = 1u << wd.wpr_lg, tile = blockIdx.x;
  uint32_t* cnt = osm; uint32_t* lbase = cnt + wpr; uint32_t* lcur = lbase + wpr; uint32_t* gbase = lcur + wpr;
  uint32_t* stage = gbase + wpr;
  __shared__ uint32_t warp_tot[32];
  __shared__ uint32_t s_chunk[OLD_UNITS], s_n[OLD_UNITS];
  __shared__ uint32_t s_skip;
  const uint32_t tid = threadIdx.x;
  for(uint32_t i = tid; i < wpr; i += 1024) cnt[i] = 0;
  uint32_t r = 0;
  while(r + 1 < wd.G && wd.stile_first[r + 1] <= tile) ++r;
  const uint32_t u0 = wd.unit_first[r] + (tile - wd.stile_first[r]) * OLD_UNITS;
  const uint32_t u1 = min(u0 + OLD_UNITS, wd.unit_first[r + 1]);
  if(tid < OLD_UNITS) {
    uint32_t c = 0, n = 0;
    if(u0 + tid < u1) { c = __ldg(order + u0 + tid); n = __ldg(&pd.dir[c].y); }
    s_chunk[tid] = c; s_n[tid] = n;
  }
  __syncthreads();
  const uint32_t half = tid >> 9, piece = tid & 511u, wmask = wpr - 1;
#pragma unroll
  for(uint32_t it = 0; it < OLD_UNITS / 2; ++it) {
    const uint32_t j = 2 * it + half, n = s_n[j];
    if(piece * 4 < n) {
      const uint4 v = __ldg(reinterpret_cast<const uint4*>(pd.pool + (size_t)s_chunk[j] * CHUNK_BYTES) + piece);
      const uint32_t rec[4] = { v.x, v.y, v.z, v.w };
#pragma unroll
      for(uint32_t q = 0; q < 4; ++q) if(piece * 4 + q < n) atomicAdd(&cnt[((rec[q] >> hb) >> WIN_LG) & wmask], 1u);
    }
  }
  __syncthreads();
  const uint32_t per = (wpr + 1023) / 1024, b = tid * per;
  uint32_t s = 0;
  for(uint32_t i = b; i < min(b + per, wpr); ++i) s += cnt[i];
  uint32_t incl = s;
#pragma unroll
  for(int o = 1; o < 32; o <<= 1) { const uint32_t v = __shfl_up_sync(0xffffffffu, incl, o); if((tid & 31) >= (uint32_t)o) incl += v; }
  if((tid & 31) == 31) warp_tot[tid >> 5] = incl;
  __syncthreads();
  uint32_t woff = 0, total = 0;
  for(uint32_t w = 0; w < 32; ++w) { const uint32_t x = warp_tot[w]; if(w < (tid >> 5)) woff += x; total += x; }
  uint32_t run = woff + incl - s;
  for(uint32_t i = b; i < min(b + per, wpr); ++i) {
    const uint32_t c = cnt[i];
    lbase[i] = run; lcur[i] = run;
    uint32_t at = 0;
    if(c) {
      const uint32_t gw = (r << wd.wpr_lg) + i;
      at = atomicAdd(&wd.wcursor[gw], c);
      if(at + c <= wd.cap) at += gw * wd.cap;
      else { at = (uint32_t)wd.wrec_cap; *(volatile uint32_t*)wd.overflow = 1u; }
    }
    gbase[i] = at - run;
    run += c;
  }
  if(tid == 0) s_skip = *(volatile uint32_t*)wd.overflow;
  __syncthreads();
  if(s_skip) return;
#pragma unroll
  for(uint32_t it = 0; it < OLD_UNITS / 2; ++it) {
    const uint32_t j = 2 * it + half, n = s_n[j];
    if(piece * 4 < n) {
      const uint4 v = __ldcs(reinterpret_cast<const uint4*>(pd.pool + (size_t)s_chunk[j] * CHUNK_BYTES) + piece);
      const uint32_t rec[4] = { v.x, v.y, v.z, v.w };
#pragma unroll
      for(uint32_t q = 0; q < 4; ++q) if(piece * 4 + q < n) stage[atomicAdd(&lcur[((rec[q] >> hb) >> WIN_LG) & wmask], 1u)] = rec[q];
    }
  }
  __syncthreads();
  for(uint32_t i = tid; i < total; i += 1024) {
    const uint32_t v = stage[i], w = ((v >> hb) >> WIN_LG) & wmask;
    const uint32_t dst = gbase[w] + i;
    if(dst < wd.wrec_cap) wd.wrec[dst] = v;
  }
}

template<uint32_t UNITS, uint32_t NBUF, uint32_t NTH>
__global__ void __launch_bounds__(NTH, 1) tiles_kernel(PartDev pd, WinDev wd, const uint32_t* __restrict__ order, uint32_t hb) {
  win_scatter_tiles<true, UNITS, NBUF, NTH>(pd, wd, order, hb);
}

struct Setup {
  uint32_t G = 12, region_bits = 23, wpr_lg = 9, hb = 9, chunks_per_region = 2384;
  uint32_t n_chunks = 0; uint64_t n_recs = 0;
  std::vector<uint32_t> order, dir_n, pool;     // host copies
  std::vector<uint64_t> win_cnt, win_sum;      // per window of the group: records, sum of records
  uint8_t* d_pool = nullptr; uint2* d_dir = nullptr; uint32_t* d_order = nullptr;
  uint32_t *d_wcursor = nullptr, *d_wrec = nullptr, *d_flag = nullptr;
  uint64_t wrec_cap = (uint64_t)64 << 20, cap = 0;
};

static WinDev make_wd(const Setup& S, uint32_t units) {
  WinDev wd; memset(&wd, 0, sizeof(wd));
  uint32_t tiles = 0;
  for(uint32_t r = 0; r < S.G; ++r) {
    wd.stile_first[r] = tiles; wd.unit_first[r] = r * S.chunks_per_region;
    tiles += (S.chunks_per_region + units - 1) / units;
  }
  wd.stile_first[S.G] = tiles; wd.unit_first[S.G] = S.G * S.chunks_per_region;
  wd.g0 = 0; wd.G = S.G; wd.wpr_lg = S.wpr_lg; wd.n_tiles = tiles; wd.cap = (uint32_t)S.cap;
  wd.overflow = S.d_flag; wd.wcursor = S.d_wcursor; wd.wrec = S.d_wrec; wd.wrec_cap = S.wrec_cap;
  return wd;
}

static bool check(const Setup& S, const char* name) {
  const uint32_t n_win = S.G << S.wpr_lg;
  std::vector<uint32_t> cur(n_win), rec((size_t)n_win * S.cap);
  uint32_t flag = 0;
  CK(cudaMemcpy(cur.data(), S.d_wcursor, n_win * 4, cudaMemcpyDeviceToHost));
  CK(cudaMemcpy(rec.data(), S.d_wrec, rec.size() * 4, cudaMemcpyDeviceToHost));
  CK(cudaMemcpy(&flag, S.d_flag, 4, cudaMemcpyDeviceToHost));
  if(flag) { printf("%s: a bucket overflowed\n", name); return false; }
  for(uint32_t w = 0; w < n_win; ++w) {
    uint64_t sum = 0;
    for(uint32_t i = 0; i < cur[w]; ++i) {
      const uint32_t v = rec[(size_t)w * S.cap + i];
      if((((v >> S.hb) >> WIN_LG) & ((1u << S.wpr_lg) - 1)) != (w & ((1u << S.wpr_lg) - 1))) { printf("%s: window %u holds a foreign record\n", name, w); return false; }
      sum += v;
    }
    if(cur[w] != S.win_cnt[w] || sum != S.win_sum[w]) { printf("%s: window %u: %u records (expected %llu)\n", name, w, cur[w], (unsigned long long)S.win_cnt[w]); return false; }
  }
  return true;
}

static std::string smi() {
  std::string out;
  if(FILE* f = popen("nvidia-smi --query-gpu=name,power.limit,clocks.sm,clocks.max.sm,clocks_throttle_reasons.active --format=csv,noheader 2>/dev/null", "r")) {
    char buf[512]; while(fgets(buf, sizeof buf, f)) out += buf;
    pclose(f);
  }
  while(!out.empty() && (out.back() == '\n' || out.back() == '\r')) out.pop_back();
  return out;
}

int main(int argc, char** argv) {
  const int iters = argc > 1 ? atoi(argv[1]) : 50;
  Setup S;
  uint32_t partial_every = 64;                  // one chunk in this many holds fewer than 2048 records
  if(argc > 5) {                                // another geometry: windows per region (log2), regions, chunks per region, partial_every
    S.wpr_lg = atoi(argv[2]); S.G = atoi(argv[3]); S.chunks_per_region = atoi(argv[4]); partial_every = atoi(argv[5]);
    S.region_bits = WIN_LG + S.wpr_lg; S.hb = 32 - S.region_bits;
  }
  int n_sm = 0; CK(cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, 0));
  const uint32_t CR = CHUNK_BYTES / 4, wpr = 1u << S.wpr_lg;
  S.n_chunks = S.G * S.chunks_per_region;
  // chunks of every region full, except one in 64 that holds a random number of records (the chunks K1 left open)
  std::mt19937_64 rng(12345);
  S.order.resize(S.n_chunks); S.dir_n.resize(S.n_chunks); S.pool.assign((size_t)S.n_chunks * CR, 0);
  std::vector<uint32_t> perm(S.n_chunks);
  for(uint32_t i = 0; i < S.n_chunks; ++i) perm[i] = i;
  std::shuffle(perm.begin(), perm.end(), rng);
  S.win_cnt.assign(S.G << S.wpr_lg, 0); S.win_sum.assign(S.G << S.wpr_lg, 0);
  uint64_t max_region = 0;
  for(uint32_t r = 0; r < S.G; ++r) {
    uint64_t in_region = 0;
    for(uint32_t u = 0; u < S.chunks_per_region; ++u) {
      const uint32_t c = perm[r * S.chunks_per_region + u];
      const uint32_t n = rng() % partial_every == 0 ? (uint32_t)(rng() % CR) + 1 : CR;
      S.order[r * S.chunks_per_region + u] = c; S.dir_n[c] = n;
      for(uint32_t i = 0; i < n; ++i) {
        const uint32_t v = (uint32_t)(rng() >> 32);
        S.pool[(size_t)c * CR + i] = v;
        const uint32_t w = (r << S.wpr_lg) + (((v >> S.hb) >> WIN_LG) & (wpr - 1));
        S.win_cnt[w] += 1; S.win_sum[w] += v;
      }
      in_region += n;
    }
    S.n_recs += in_region; max_region = std::max(max_region, in_region);
  }
  const uint64_t m = (max_region + wpr - 1) / wpr;          // the engine's bucket capacity rule (jf_engine.cu, bucket_cap)
  S.cap = (m + (uint64_t)std::ceil(6.0 * std::sqrt((double)m)) + 16 + 3) & ~(uint64_t)3;
  std::vector<uint2> dir(S.n_chunks);
  for(uint32_t c = 0; c < S.n_chunks; ++c) dir[c] = make_uint2(0, S.dir_n[c]);
  CK(cudaMalloc(&S.d_pool, (size_t)S.n_chunks * CHUNK_BYTES)); CK(cudaMalloc(&S.d_dir, S.n_chunks * 8)); CK(cudaMalloc(&S.d_order, S.n_chunks * 4));
  CK(cudaMalloc(&S.d_wcursor, (S.G << S.wpr_lg) * 4)); CK(cudaMalloc(&S.d_wrec, S.wrec_cap * 4 + 64)); CK(cudaMalloc(&S.d_flag, 4));
  CK(cudaMemcpy(S.d_pool, S.pool.data(), (size_t)S.n_chunks * CHUNK_BYTES, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(S.d_dir, dir.data(), S.n_chunks * 8, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(S.d_order, S.order.data(), S.n_chunks * 4, cudaMemcpyHostToDevice));
  PartDev pd; memset(&pd, 0, sizeof(pd));
  pd.region_bits = S.region_bits; pd.rec_bytes = 4; pd.chunk_recs = CR; pd.n_chunks = S.n_chunks; pd.pool = S.d_pool; pd.dir = S.d_dir;

  cudaEvent_t a, b; CK(cudaEventCreate(&a)); CK(cudaEventCreate(&b));
  const double bytes = 8.0 * (double)S.n_recs;
  printf("{\"bench\": \"win_scatter\", \"gpu\": \"%s\", \"regions\": %u, \"partial_every\": %u, \"windows_per_region\": %u, \"records\": %llu, \"bucket_cap\": %llu, \"launches\": %d}\n",
         smi().c_str(), S.G, partial_every, wpr, (unsigned long long)S.n_recs, (unsigned long long)S.cap, iters);
  auto report = [&](const char* name, uint32_t units, double ms_per, bool ok) {
    const double runs = units ? (double)S.n_recs / ((double)S.G * ((S.chunks_per_region + units - 1) / units) * wpr) : 0;
    printf("  %-40s %8.3f ms  %6.2f G records/s  %7.1f GB/s  mean run %5.1f records  %s\n", name, ms_per, S.n_recs / ms_per / 1e6,
           bytes / ms_per / 1e6, runs, ok ? "buckets ok" : "BUCKETS WRONG");
  };
  // one form: a checked launch, then `iters` timed launches (wcursor and the flag cleared before each, outside the events)
  auto timed = [&](const char* name, uint32_t units, auto launch) {
    CK(cudaMemset(S.d_wcursor, 0, (S.G << S.wpr_lg) * 4)); CK(cudaMemset(S.d_flag, 0, 4)); CK(cudaMemset(S.d_wrec, 0xFF, S.wrec_cap * 4));
    launch(); CK(cudaGetLastError()); CK(cudaDeviceSynchronize());
    const bool ok = check(S, name);
    double total = 0;
    for(int i = 0; i < iters; ++i) {
      CK(cudaMemsetAsync(S.d_wcursor, 0, (S.G << S.wpr_lg) * 4)); CK(cudaMemsetAsync(S.d_flag, 0, 4));
      CK(cudaEventRecord(a)); launch(); CK(cudaEventRecord(b)); CK(cudaEventSynchronize(b));
      float ms = 0; CK(cudaEventElapsedTime(&ms, a, b)); total += ms;
    }
    report(name, units, total / iters, ok);
  };
  auto new_form = [&](const char* name, auto kern, uint32_t units, uint32_t nbuf, uint32_t nth) {
    const WinDev wd = make_wd(S, units);
    const size_t smem = win_scatter_smem(units, nbuf, wpr);
    CK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    timed(name, units, [&] { kern<<<std::min<uint32_t>(wd.n_tiles, n_sm), nth, smem>>>(pd, wd, S.d_order, S.hb); });
  };
  {
    // the exact pass (win_scatter_kernel<false>): the flag set from the start, so the bucket pass only counts; the run
    // starts are the scan of the counts (each rounded up to 4 records), as win_scan_kernel makes them
    const WinDev wd = make_wd(S, WIN_ST_UNITS);
    const size_t smem = win_scatter_smem(WIN_ST_UNITS, WIN_ST_NBUF, wpr);
    const uint32_t n_win = S.G << S.wpr_lg, grid = std::min<uint32_t>(wd.n_tiles, n_sm);
    CK(cudaFuncSetAttribute(win_scatter_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    CK(cudaFuncSetAttribute(win_scatter_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const uint32_t one = 1;
    CK(cudaMemset(S.d_wcursor, 0, n_win * 4)); CK(cudaMemcpy(S.d_flag, &one, 4, cudaMemcpyHostToDevice));
    win_scatter_kernel<true><<<grid, WIN_ST_NTH, smem>>>(pd, wd, S.d_order, S.hb); CK(cudaGetLastError());
    std::vector<uint32_t> cur(n_win), start(n_win);
    CK(cudaMemcpy(cur.data(), S.d_wcursor, n_win * 4, cudaMemcpyDeviceToHost));
    bool ok = true;
    uint32_t at = 0;
    for(uint32_t w = 0; w < n_win; ++w) { ok &= cur[w] == S.win_cnt[w]; start[w] = at; at += (cur[w] + 3) & ~3u; }
    CK(cudaMemcpy(S.d_wcursor, start.data(), n_win * 4, cudaMemcpyHostToDevice));
    CK(cudaMemset(S.d_wrec, 0xFF, S.wrec_cap * 4));
    win_scatter_kernel<false><<<grid, WIN_ST_NTH, smem>>>(pd, wd, S.d_order, S.hb); CK(cudaGetLastError());
    std::vector<uint32_t> rec(at);
    CK(cudaMemcpy(rec.data(), S.d_wrec, (size_t)at * 4, cudaMemcpyDeviceToHost));
    for(uint32_t w = 0; w < n_win && ok; ++w) {
      uint64_t sum = 0;
      for(uint32_t i = 0; i < cur[w]; ++i) {
        const uint32_t v = rec[start[w] + i];
        ok &= (((v >> S.hb) >> WIN_LG) & (wpr - 1)) == (w & (wpr - 1));
        sum += v;
      }
      ok &= sum == S.win_sum[w];
    }
    printf("  exact pass (win_scatter_kernel<false>, %u chunks x %u buffers, %u threads): %s\n", WIN_ST_UNITS, WIN_ST_NBUF, WIN_ST_NTH, ok ? "runs ok" : "RUNS WRONG");
  }
  for(int rep = 0; rep < 2; ++rep) {
    {
      const WinDev wd = make_wd(S, OLD_UNITS);
      const size_t smem = ((size_t)4 * wpr + (size_t)OLD_UNITS * CR) * 4;
      CK(cudaFuncSetAttribute(old_scatter_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
      timed("previous: 12 chunks, CTA per tile", OLD_UNITS, [&] { old_scatter_kernel<<<wd.n_tiles, 1024, smem>>>(pd, wd, S.d_order, S.hb); });
    }
    new_form("persistent: 12 chunks x 2, 768 threads", tiles_kernel<12, 2, 768>, 12, 2, 768);
    new_form("persistent: 12 chunks x 2, 512 threads", tiles_kernel<12, 2, 512>, 12, 2, 512);
    new_form("persistent: 12 chunks x 2, 1024 threads", tiles_kernel<12, 2, 1024>, 12, 2, 1024);
    new_form("persistent: 8 chunks x 3, 1024 threads", tiles_kernel<8, 3, 1024>, 8, 3, 1024);
    new_form("persistent: 8 chunks x 2, 1024 threads", tiles_kernel<8, 2, 1024>, 8, 2, 1024);
    new_form("persistent: 4 chunks x 3, 1024 threads", tiles_kernel<4, 3, 1024>, 4, 3, 1024);
    {
      double total = 0;
      for(int i = 0; i < iters; ++i) {
        CK(cudaEventRecord(a)); CK(cudaMemcpyAsync(S.d_wrec, S.d_pool, S.n_recs * 4, cudaMemcpyDeviceToDevice)); CK(cudaEventRecord(b));
        CK(cudaEventSynchronize(b)); float ms = 0; CK(cudaEventElapsedTime(&ms, a, b)); total += ms;
      }
      report("cudaMemcpy of the same bytes (ceiling)", 0, total / iters, true);
    }
  }
  printf("{\"gpu_after\": \"%s\"}\n", smi().c_str());
  return 0;
}
