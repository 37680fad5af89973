// The window form of K2 (jf_window.cuh) behind a small C ABI, so that tests/test_gpu_win_kernels.py can launch its kernels
// directly on inputs built to hit one edge each and judge them with the exact models of tests/win_model.py.
//
//   win_harness_place   the bucket pass (K2b, win_scatter_kernel<true>), win_scan_kernel and the exact pass (K2a,
//                       win_scatter_kernel<false>) of one group, launched as part_drain launches them (jf_engine.cu)
//   win_harness_insert  win_insert2_kernel<1> (K2c), win_zero_kernel when the drain is write-only, win_deferred_kernel<1>
//
// Every entry point takes host arrays, allocates, copies, launches, synchronises, copies back and frees.  It returns 0, or
// 1 with a message when an input breaks a precondition the kernels rely on (those are checked before anything is launched,
// since a broken one means an access out of bounds), or 2 with the CUDA error.  The kernels are compiled from the
// engine's sources in this translation unit, with the library's flags:
//
//   nvcc -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a --expt-relaxed-constexpr -Xcompiler -fPIC -shared \
//        -I jellyfish_b200/csrc -o win_harness.so tests/win_harness.cu
#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <vector>
#include "jf_kernels.cuh"
#include "jf_window.cuh"

using namespace jfk;

namespace {

struct Call {                                      // the device buffers of one call, freed when it returns
  std::vector<void*> bufs;
  char* err; size_t err_len;
  ~Call() { for(void* p : bufs) cudaFree(p); }
  template<class T> cudaError_t alloc(T*& p, size_t n) {
    void* q = nullptr;
    const cudaError_t e = cudaMalloc(&q, n * sizeof(T) + 64);
    if(e == cudaSuccess) { bufs.push_back(q); p = static_cast<T*>(q); }
    return e;
  }
  int refuse(const char* msg) { snprintf(err, err_len, "%s", msg); return 1; }
  int cuda(const char* what, cudaError_t e) { snprintf(err, err_len, "%s: %s", what, cudaGetErrorString(e)); return 2; }
};

#define HCK(x) do { const cudaError_t e_ = (x); if(e_ != cudaSuccess) return call.cuda(#x, e_); } while(0)
#define NEED(c, msg) do { if(!(c)) return call.refuse(msg); } while(0)

int n_sm_of_device() {
  int n = 0;
  return cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, 0) == cudaSuccess ? n : 0;
}

}  // namespace

extern "C" int win_harness_n_sm() { return n_sm_of_device(); }

// One group of G regions [g0, g0 + G) with 2^wpr_lg windows each.  pool: n_chunks chunks of CHUNK_BYTES; dir_n: records of
// every chunk; order: the units (chunk ids) in region order, region r's at [unit_first[r], unit_first[r + 1]).  flag0: the
// group's overflow flag before the bucket pass (1 as part_drain sets it for k2_mode 3).
// Out: the flag, wcursor after the bucket pass, wstart [n + 1], wcnt [n], wrec [0, wrec_n) (wrec_n <= wrec_cap), the
// STAT_POOL_FULL count, with n = G << wpr_lg.  wrec is filled with `fill` before the bucket pass.
extern "C" int win_harness_place(const uint32_t* pool, uint32_t n_chunks, const uint32_t* dir_n, const uint32_t* order, uint32_t n_order,
                                 const uint32_t* unit_first, uint32_t g0, uint32_t G, uint32_t wpr_lg, uint32_t hb, uint32_t cap,
                                 uint64_t wrec_cap, uint32_t flag0, uint32_t fill,
                                 uint32_t* flag_out, uint32_t* wcursor_out, uint32_t* wstart_out, uint32_t* wcnt_out, uint32_t* wrec_out,
                                 uint64_t wrec_n, unsigned long long* pool_full_out, char* err, size_t err_len) {
  Call call{{}, err, err_len};
  NEED(G >= 1 && G <= WIN_MAX_G, "G out of 1..64");
  NEED(wpr_lg >= 1 && wpr_lg <= 11, "wpr_lg out of 1..11");
  NEED(hb + WIN_LG + wpr_lg <= 32, "hb + region_bits > 32");
  NEED(cap > 0 && cap % 4 == 0, "cap must be a positive multiple of 4 (buckets start on 16-byte boundaries)");
  const uint32_t n = G << wpr_lg;
  NEED((uint64_t)n * cap <= 0xFFFFFFFFull && wrec_cap <= 0xFFFFFFFFull && wrec_cap >= (uint64_t)n * cap, "wrec_cap out of n * cap .. 2^32 - 1");
  NEED(wrec_n <= wrec_cap, "wrec_n > wrec_cap");
  NEED(unit_first[G] <= n_order, "unit_first[G] > n_order");
  uint32_t stiles = 0;
  std::vector<uint32_t> stile_first(G + 1);
  for(uint32_t r = 0; r < G; ++r) {
    NEED(unit_first[r] <= unit_first[r + 1], "unit_first must not decrease");
    stile_first[r] = stiles;
    stiles += (unit_first[r + 1] - unit_first[r] + WIN_ST_UNITS - 1) / WIN_ST_UNITS;
  }
  stile_first[G] = stiles;
  for(uint32_t u = unit_first[0]; u < unit_first[G]; ++u) NEED(order[u] < n_chunks, "order names a chunk past the pool");
  for(uint32_t c = 0; c < n_chunks; ++c) NEED(dir_n[c] <= CHUNK_BYTES / 4, "a chunk holds more than 2048 records");
  const int n_sm = n_sm_of_device();
  NEED(n_sm > 0, "no CUDA device");

  uint8_t* d_pool; uint2* d_dir; uint32_t *d_order, *d_flag, *d_wstart, *d_wcursor, *d_wcnt, *d_wrec; unsigned long long* d_stats;
  HCK(call.alloc(d_pool, (size_t)n_chunks * CHUNK_BYTES)); HCK(call.alloc(d_dir, n_chunks)); HCK(call.alloc(d_order, n_order));
  HCK(call.alloc(d_flag, 1)); HCK(call.alloc(d_wstart, n + 1)); HCK(call.alloc(d_wcursor, n)); HCK(call.alloc(d_wcnt, n));
  HCK(call.alloc(d_wrec, wrec_cap)); HCK(call.alloc(d_stats, STAT_N));        // (alloc adds the engine's 64 bytes of slack)
  std::vector<uint2> dir(n_chunks);
  for(uint32_t c = 0; c < n_chunks; ++c) dir[c] = make_uint2(0, dir_n[c]);
  HCK(cudaMemcpy(d_pool, pool, (size_t)n_chunks * CHUNK_BYTES, cudaMemcpyHostToDevice));
  HCK(cudaMemcpy(d_dir, dir.data(), (size_t)n_chunks * sizeof(uint2), cudaMemcpyHostToDevice));
  HCK(cudaMemcpy(d_order, order, (size_t)n_order * 4, cudaMemcpyHostToDevice));
  HCK(cudaMemcpy(d_flag, &flag0, 4, cudaMemcpyHostToDevice));
  HCK(cudaMemset(d_wcursor, 0, (size_t)n * 4));
  HCK(cudaMemset(d_stats, 0, STAT_N * 8));
  {
    std::vector<uint32_t> f(wrec_cap + 16, fill);
    HCK(cudaMemcpy(d_wrec, f.data(), f.size() * 4, cudaMemcpyHostToDevice));
  }

  PartDev pd; memset(&pd, 0, sizeof(pd));
  pd.region_bits = WIN_LG + wpr_lg; pd.rec_bytes = 4; pd.chunk_recs = CHUNK_BYTES / 4; pd.n_chunks = n_chunks;
  pd.pool = d_pool; pd.dir = d_dir;
  WinDev wd; memset(&wd, 0, sizeof(wd));
  for(uint32_t r = 0; r <= G; ++r) { wd.stile_first[r] = stile_first[r]; wd.unit_first[r] = unit_first[r]; }
  wd.g0 = g0; wd.G = G; wd.wpr_lg = wpr_lg; wd.n_tiles = stiles; wd.cap = cap;
  wd.overflow = d_flag; wd.wstart = d_wstart; wd.wcursor = d_wcursor; wd.wcnt = d_wcnt; wd.wrec = d_wrec; wd.wrec_cap = wrec_cap;

  const size_t smem = win_scatter_smem(WIN_ST_UNITS, WIN_ST_NBUF, 1u << wpr_lg);
  HCK(cudaFuncSetAttribute(win_scatter_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  HCK(cudaFuncSetAttribute(win_scatter_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const uint32_t grid = std::min<uint32_t>(stiles, (uint32_t)n_sm);
  if(grid) {                                       // (part_drain launches nothing for a group without tiles)
    win_scatter_kernel<true><<<grid, WIN_ST_NTH, smem>>>(pd, wd, d_order, hb);
    HCK(cudaGetLastError()); HCK(cudaDeviceSynchronize());
    HCK(cudaMemcpy(wcursor_out, d_wcursor, (size_t)n * 4, cudaMemcpyDeviceToHost));
    win_scan_kernel<<<1, 1024>>>(wd, d_stats);
    HCK(cudaGetLastError());
    win_scatter_kernel<false><<<grid, WIN_ST_NTH, smem>>>(pd, wd, d_order, hb);
    HCK(cudaGetLastError()); HCK(cudaDeviceSynchronize());
  } else {
    memset(wcursor_out, 0, (size_t)n * 4);
    HCK(cudaMemset(d_wstart, 0, (size_t)(n + 1) * 4)); HCK(cudaMemset(d_wcnt, 0, (size_t)n * 4));
  }
  HCK(cudaMemcpy(flag_out, d_flag, 4, cudaMemcpyDeviceToHost));
  HCK(cudaMemcpy(wstart_out, d_wstart, (size_t)(n + 1) * 4, cudaMemcpyDeviceToHost));
  HCK(cudaMemcpy(wcnt_out, d_wcnt, (size_t)n * 4, cudaMemcpyDeviceToHost));
  HCK(cudaMemcpy(wrec_out, d_wrec, wrec_n * 4, cudaMemcpyDeviceToHost));
  HCK(cudaMemcpy(pool_full_out, d_stats + STAT_POOL_FULL, 8, cudaMemcpyDeviceToHost));
  return 0;
}

// One drain of group [g0, g0 + G) into a table of 2^local_lsize 32-bit slots (one shard) plus the margin: `table` holds
// local_size + tri(max_reprobe) + 8 slots, in and out.  win_state: the table's window states (local_size >> WIN_LG of them)
// for a write-only drain, else null.  wstart/wcnt [G << wpr_lg] and wrec [wrec_n] as win_scan leaves them (either layout).
// ovf_keys/ovf_vals [ovf_size]: the counter-carry side table, in and out.  Out: the STAT_N statistics and the number of
// deferred records.
extern "C" int win_harness_insert(uint32_t* table, uint32_t local_lsize, uint32_t fbits, uint32_t rbits, uint32_t max_reprobe,
                                  const uint32_t* win_state, uint32_t g0, uint32_t G, uint32_t wpr_lg,
                                  const uint32_t* wstart, const uint32_t* wcnt, const uint32_t* wrec, uint64_t wrec_n,
                                  uint64_t* ovf_keys, uint64_t* ovf_vals, uint64_t ovf_size,
                                  unsigned long long* stats_out, unsigned long long* def_n_out, char* err, size_t err_len) {
  Call call{{}, err, err_len};
  NEED(G >= 1 && G <= WIN_MAX_G, "G out of 1..64");
  NEED(wpr_lg >= 1 && wpr_lg <= 11, "wpr_lg out of 1..11");
  const uint32_t region_bits = WIN_LG + wpr_lg;
  NEED(local_lsize >= region_bits && local_lsize <= 34, "local_lsize out of region_bits..34");
  const uint64_t local_size = (uint64_t)1 << local_lsize;
  NEED(((uint64_t)(g0 + G) << region_bits) <= local_size, "the group reaches past the table");
  NEED(rbits >= 1 && rbits <= 8 && ((max_reprobe + 1) >> rbits) == 0, "the reprobe field cannot hold max_reprobe + 1");
  NEED(fbits >= rbits && fbits <= 22, "fbits out of rbits..22");
  NEED(max_reprobe >= 1 && tri(max_reprobe) < ((uint64_t)1 << region_bits), "tri(max_reprobe) must stay inside a region");
  NEED(ovf_size >= 1024 && (ovf_size & (ovf_size - 1)) == 0, "ovf_size must be a power of two >= 1024");
  const uint32_t n = G << wpr_lg;
  uint64_t total = 0;
  for(uint32_t i = 0; i < n; ++i) {
    NEED(wstart[i] % 4 == 0, "a run does not start on a 16-byte boundary");
    NEED((uint64_t)wstart[i] + wcnt[i] <= wrec_n, "a run reaches past wrec");
    total += wcnt[i];
  }
  const int n_sm = n_sm_of_device();
  NEED(n_sm > 0, "no CUDA device");
  const uint64_t n_slots = local_size + tri(max_reprobe) + 8;
  const uint32_t nbytes = 8;                       // (one-word keys: the inverse tables k2_fail reads, as table_setup sizes them)

  uint32_t *d_tab, *d_state = nullptr, *d_wstart, *d_wcnt, *d_wrec, *d_def_high;
  uint64_t *d_inv, *d_def_pos, *d_fail_keys, *d_fail_counts;
  unsigned long long *d_ovf_keys, *d_ovf_vals, *d_stats, *d_def_n;
  const uint64_t def_cap = total + 1, fail_cap = total + 1;
  HCK(call.alloc(d_tab, n_slots)); HCK(call.alloc(d_wstart, n + 1)); HCK(call.alloc(d_wcnt, n)); HCK(call.alloc(d_wrec, wrec_n));
  HCK(call.alloc(d_inv, (size_t)nbytes * 256)); HCK(call.alloc(d_def_pos, def_cap)); HCK(call.alloc(d_def_high, def_cap));
  HCK(call.alloc(d_fail_keys, fail_cap)); HCK(call.alloc(d_fail_counts, fail_cap));
  HCK(call.alloc(d_ovf_keys, ovf_size)); HCK(call.alloc(d_ovf_vals, ovf_size)); HCK(call.alloc(d_stats, STAT_N)); HCK(call.alloc(d_def_n, 1));
  if(win_state) {
    HCK(call.alloc(d_state, local_size >> WIN_LG));
    HCK(cudaMemcpy(d_state, win_state, (local_size >> WIN_LG) * 4, cudaMemcpyHostToDevice));
  }
  HCK(cudaMemcpy(d_tab, table, n_slots * 4, cudaMemcpyHostToDevice));
  HCK(cudaMemcpy(d_wstart, wstart, (size_t)n * 4, cudaMemcpyHostToDevice));
  HCK(cudaMemcpy(d_wcnt, wcnt, (size_t)n * 4, cudaMemcpyHostToDevice));
  HCK(cudaMemset(d_wrec, 0, wrec_n * 4 + 64));
  HCK(cudaMemcpy(d_wrec, wrec, wrec_n * 4, cudaMemcpyHostToDevice));
  HCK(cudaMemset(d_inv, 0, (size_t)nbytes * 256 * 8));
  HCK(cudaMemcpy(d_ovf_keys, ovf_keys, ovf_size * 8, cudaMemcpyHostToDevice));
  HCK(cudaMemcpy(d_ovf_vals, ovf_vals, ovf_size * 8, cudaMemcpyHostToDevice));
  HCK(cudaMemset(d_stats, 0, STAT_N * 8)); HCK(cudaMemset(d_def_n, 0, 8));

  TableDev T; memset(&T, 0, sizeof(T));
  T.slots = d_tab; T.local_mask = local_size - 1; T.local_lsize = local_lsize; T.lsize = local_lsize; T.shard_index = 0;
  T.kbits = 8 * nbytes; T.rbits = rbits; T.fbits = fbits; T.max_reprobe = max_reprobe; T.op = 0;
  T.ovf_keys = d_ovf_keys; T.ovf_vals = d_ovf_vals; T.ovf_mask = ovf_size - 1; T.stats = d_stats;
  T.fail_keys = d_fail_keys; T.fail_counts = d_fail_counts; T.fail_cap = fail_cap;
  PartDev pd; memset(&pd, 0, sizeof(pd));
  pd.region_bits = region_bits; pd.rec_bytes = 4; pd.chunk_recs = CHUNK_BYTES / 4;
  WinDev wd; memset(&wd, 0, sizeof(wd));
  wd.g0 = g0; wd.G = G; wd.wpr_lg = wpr_lg; wd.lazy_win = d_state;
  wd.wstart = d_wstart; wd.wcnt = d_wcnt; wd.wrec = d_wrec; wd.wrec_cap = wrec_n;
  wd.def_pos = d_def_pos; wd.def_high = d_def_high; wd.def_n = d_def_n; wd.def_cap = def_cap;

  HCK(cudaFuncSetAttribute(win_insert2_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)WIN2_SMEM));
  win_insert2_kernel<1><<<n_sm, WIN2_NTH, WIN2_SMEM>>>(T, pd, wd, d_inv, nbytes);
  HCK(cudaGetLastError());
  if(d_state) {
    win_zero_kernel<<<n_sm * 4, 256>>>(d_tab, d_state, d_wcnt, (uint64_t)g0 << wpr_lg, n);
    HCK(cudaGetLastError());
  }
  win_deferred_kernel<1><<<n_sm * 2, 256>>>(T, wd, d_inv, nbytes);
  HCK(cudaGetLastError()); HCK(cudaDeviceSynchronize());
  HCK(cudaMemcpy(table, d_tab, n_slots * 4, cudaMemcpyDeviceToHost));
  HCK(cudaMemcpy(ovf_keys, d_ovf_keys, ovf_size * 8, cudaMemcpyDeviceToHost));
  HCK(cudaMemcpy(ovf_vals, d_ovf_vals, ovf_size * 8, cudaMemcpyDeviceToHost));
  HCK(cudaMemcpy(stats_out, d_stats, STAT_N * 8, cudaMemcpyDeviceToHost));
  HCK(cudaMemcpy(def_n_out, d_def_n, 8, cudaMemcpyDeviceToHost));
  return 0;
}
