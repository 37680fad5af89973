// jf_query.cuh -- the kernels of `query -s` and of loading a database back into a table.
//
//   Q0 query_decode_kernel  binary/sorted record bytes -> key words + counts (then insert_keys_kernel, K2')
//   Q1 extract_kernel MODE 3 (jf_extract.cuh): the k-mers of every window in input order, q_cnt[t] of them
//   Q2 query_lookup_kernel  one CTA per window: count of every k-mer (table_get, the probe loop of lookup_kernel) and the
//                           bytes of the window's output lines
//   Q3 query_scan_kernel    exclusive scan of those byte counts (one CTA): where each window's lines start
//   Q4 query_format_kernel  one CTA per window: the lines "MER COUNT\n" (query_main.cc:45-51), in input order
#ifndef JF_QUERY_CUH
#define JF_QUERY_CUH
#include "jf_kernels.cuh"

namespace jfk {

constexpr uint32_t QUERY_NTH = 256;

// binary_reader::next (binary_dumper.hpp:103-108): key_bytes little-endian key bytes, then ocl count bytes
template<int KW>
__global__ void __launch_bounds__(256) query_decode_kernel(const uint8_t* __restrict__ rec, uint64_t n, uint32_t key_bytes, uint32_t ocl,
                                                           uint64_t* __restrict__ keys, uint64_t* __restrict__ counts) {
  const uint32_t rb = key_bytes + ocl;
  for(uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
    const uint8_t* p = rec + i * rb;
    uint64_t w[KW > 2 ? 4 : 2] = { 0, 0 }, c = 0;
    for(uint32_t b = 0; b < key_bytes; ++b) w[b >> 3] |= (uint64_t)p[b] << (8 * (b & 7));
    for(uint32_t b = 0; b < ocl; ++b) c |= (uint64_t)p[key_bytes + b] << (8 * b);
#pragma unroll
    for(int q = 0; q < KW; ++q) keys[i * KW + q] = w[q];
    counts[i] = c;
  }
}

__device__ __forceinline__ uint32_t dec_digits(uint64_t v) { uint32_t d = 1; while(v >= 10) { v /= 10; ++d; } return d; }

template<int KW, int SB>
__global__ void __launch_bounds__(QUERY_NTH) query_lookup_kernel(TableDev T, const uint64_t* __restrict__ lut_g, uint32_t nbytes,
                                                                 const uint64_t* __restrict__ keys, const uint32_t* __restrict__ cnt,
                                                                 uint32_t tile_cap, uint64_t n_tiles, uint32_t k, uint32_t shard_bits,
                                                                 uint64_t* __restrict__ vals, unsigned long long* __restrict__ tile_bytes) {
  extern __shared__ __align__(16) uint8_t smem_raw[];
  uint64_t* lut = reinterpret_cast<uint64_t*>(smem_raw);
  __shared__ unsigned long long part[QUERY_NTH / 32];
  for(uint32_t i = threadIdx.x; i < nbytes * 256u; i += blockDim.x) lut[i] = lut_g[i];
  __syncthreads();
  for(uint64_t t = blockIdx.x; t < n_tiles; t += gridDim.x) {
    const uint64_t base = t * tile_cap;
    const uint32_t m = cnt[t];
    unsigned long long bytes = 0;
    for(uint32_t i = threadIdx.x; i < m; i += blockDim.x) {
      uint64_t key[KW];
#pragma unroll
      for(int q = 0; q < KW; ++q) key[q] = keys[(base + i) * KW + q];
      const uint64_t v = table_get<KW, SB>(T, key, gf2_hash<KW>(lut, key, (int)nbytes), shard_bits);
      vals[base + i] = v;
      bytes += k + 2 + dec_digits(v);
    }
#pragma unroll
    for(int o = 16; o; o >>= 1) bytes += __shfl_xor_sync(0xffffffffu, bytes, o);
    if((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = bytes;
    __syncthreads();
    if(threadIdx.x == 0) {
      unsigned long long s = 0;
      for(uint32_t w = 0; w < QUERY_NTH / 32; ++w) s += part[w];
      tile_bytes[t] = s;
    }
    __syncthreads();
  }
}

// in place: x[i] = x[0] + ... + x[i-1], x[n] = total (one CTA of 1024 threads, each a contiguous run of entries)
__global__ void __launch_bounds__(1024) query_scan_kernel(unsigned long long* __restrict__ x, uint64_t n) {
  __shared__ unsigned long long part[1024];
  const uint64_t per = (n + blockDim.x - 1) / blockDim.x;
  const uint64_t lo = min(n, per * threadIdx.x), hi = min(n, lo + per);
  unsigned long long s = 0;
  for(uint64_t i = lo; i < hi; ++i) s += x[i];
  part[threadIdx.x] = s;
  __syncthreads();
  if(threadIdx.x == 0) { unsigned long long run = 0; for(uint32_t i = 0; i < blockDim.x; ++i) { const unsigned long long v = part[i]; part[i] = run; run += v; } x[n] = run; }
  __syncthreads();
  unsigned long long run = part[threadIdx.x];
  for(uint64_t i = lo; i < hi; ++i) { const unsigned long long v = x[i]; x[i] = run; run += v; }
}

// The lines of window t at out + off[t] - off[first window of this piece]: the k bases (upper case, first base most
// significant, mer_dna.hpp:451-462), a space, the count in decimal, '\n'.  Rounds of QUERY_NTH lines, a block scan of their
// lengths each.
template<int KW>
__global__ void __launch_bounds__(QUERY_NTH) query_format_kernel(const uint64_t* __restrict__ keys, const uint64_t* __restrict__ vals,
                                                                 const uint32_t* __restrict__ cnt, uint32_t tile_cap, uint64_t t0, uint64_t t1,
                                                                 const unsigned long long* __restrict__ off, uint32_t k, uint8_t* __restrict__ out) {
  __shared__ uint32_t wsum[QUERY_NTH / 32];
  const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for(uint64_t t = t0 + blockIdx.x; t < t1; t += gridDim.x) {
    const uint64_t base = t * tile_cap;
    const uint32_t m = cnt[t];
    uint8_t* dst = out + (off[t] - off[t0]);
    for(uint32_t r0 = 0; r0 < m; r0 += QUERY_NTH) {
      const uint32_t i = r0 + threadIdx.x;
      const bool have = i < m;
      const uint64_t v = have ? vals[base + i] : 0;
      const uint32_t nd = dec_digits(v);
      const uint32_t len = have ? k + 2 + nd : 0;
      uint32_t inc = len;
#pragma unroll
      for(int o = 1; o < 32; o <<= 1) {
        const uint32_t up = __shfl_up_sync(0xffffffffu, inc, o);
        if(lane >= o) inc += up;
      }
      if(lane == 31) wsum[warp] = inc;
      __syncthreads();
      uint32_t before = 0, total = 0;
      for(uint32_t w = 0; w < QUERY_NTH / 32; ++w) { const uint32_t s = wsum[w]; if(w < warp) before += s; total += s; }
      __syncthreads();
      if(have) {
        uint64_t key[KW];
#pragma unroll
        for(int q = 0; q < KW; ++q) key[q] = keys[(base + i) * KW + q];
        uint8_t* p = dst + before + inc - len;
        for(uint32_t b = 0; b < k; ++b) {
          const uint32_t bit = 2 * (k - 1 - b);
          p[b] = "ACGT"[(key[KW == 1 ? 0 : (bit >> 6)] >> (bit & 63)) & 3u];
        }
        p[k] = ' ';
        uint64_t x = v;
        for(uint32_t d = nd; d; --d) { p[k + d] = (uint8_t)('0' + x % 10); x /= 10; }
        p[k + 1 + nd] = '\n';
      }
      dst += total;
    }
  }
}

}  // namespace jfk
#endif
