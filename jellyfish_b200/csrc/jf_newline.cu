// jf_newline.cu -- the newline count of jf_newline.cuh (16-byte loads, four SWAR byte compares per load) and the record-aligned
// cuts of FASTQ text.
#include "jf_newline.cuh"

namespace jfnl {
namespace {

// bytes of x equal to '\n' (exact: no carry crosses a byte)
__device__ __forceinline__ uint32_t nl_in_word(uint32_t x) {
  const uint32_t y = x ^ 0x0A0A0A0Au;                       // a '\n' byte becomes 0
  const uint32_t t = ~(((y & 0x7F7F7F7Fu) + 0x7F7F7F7Fu) | y | 0x7F7F7F7Fu);   // high bit set exactly in the zero bytes
  return __popc(t);
}

// [in, in + n): the unaligned head and tail bytes one at a time, the 16-byte aligned middle as uint4 loads (grid-stride)
__global__ void __launch_bounds__(256) count_newlines_kernel(const uint8_t* in, uint64_t n, unsigned long long* count) {
  const uint64_t head = (uint64_t)((16 - ((uintptr_t)in & 15)) & 15);
  const uint64_t h = head < n ? head : n;
  const uint64_t n_vec = (n - h) / 16;
  const uint4* v = reinterpret_cast<const uint4*>(in + h);
  const uint64_t tid = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x, stride = (uint64_t)gridDim.x * blockDim.x;
  uint32_t c = 0;
  for(uint64_t i = tid; i < n_vec; i += stride) {
    const uint4 q = __ldg(v + i);
    c += nl_in_word(q.x) + nl_in_word(q.y) + nl_in_word(q.z) + nl_in_word(q.w);
  }
  const uint64_t tail0 = h + n_vec * 16;
  if(tid < h) c += in[tid] == '\n';
  if(tid < n - tail0) c += in[tail0 + tid] == '\n';
  // warp sum, then one atomic per warp
  for(int o = 16; o > 0; o >>= 1) c += __shfl_down_sync(0xffffffffu, c, o);
  if((threadIdx.x & 31) == 0 && c) atomicAdd(count, (unsigned long long)c);
}

// ---- record-aligned cuts of FASTQ text (fastq_cuts) ----

struct FqTile { uint32_t n; int32_t last[4]; };   // newlines of a tile; last[s]: tile offset of its last '\n' whose 1-based
                                                   // index in the tile is s (mod 4), -1 when there is none

// Exclusive prefix sum over the CTA (blockDim.x a multiple of 32, at most 1024); *total gets the sum.  sm: 33 words.
__device__ __forceinline__ uint32_t block_excl_sum(uint32_t v, uint32_t* sm, uint32_t* total) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = blockDim.x >> 5;
  uint32_t x = v;
  for(int o = 1; o < 32; o <<= 1) { const uint32_t y = __shfl_up_sync(0xffffffffu, x, o); if(lane >= o) x += y; }
  __syncthreads();                          // (sm may still be read by the caller's previous use)
  if(lane == 31) sm[w] = x;
  __syncthreads();
  if(w == 0) {
    uint32_t t = lane < nw ? sm[lane] : 0, u = t;
    for(int o = 1; o < 32; o <<= 1) { const uint32_t y = __shfl_up_sync(0xffffffffu, u, o); if(lane >= o) u += y; }
    sm[lane] = u - t;
    if(lane == 31) sm[32] = u;
  }
  __syncthreads();
  *total = sm[32];
  return sm[w] + x - v;
}

// Maximum over the CTA of four values (every thread gets them).  sm: 4 * 32 long longs.
__device__ __forceinline__ void block_max4(long long v[4], long long* sm) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = blockDim.x >> 5;
  for(int s = 0; s < 4; ++s)
    for(int o = 16; o > 0; o >>= 1) v[s] = max(v[s], (long long)__shfl_xor_sync(0xffffffffu, v[s], o));
  __syncthreads();
  if(lane == 0) for(int s = 0; s < 4; ++s) sm[s * 32 + w] = v[s];
  __syncthreads();
  for(int s = 0; s < 4; ++s) {
    long long m = -1;
    for(int i = 0; i < nw; ++i) m = max(m, sm[s * 32 + i]);
    v[s] = m;
  }
}

// The newlines of bytes [o, o + 16) below `lim` (offsets relative to `base`): count and the last one of each residue of
// the running count c.
__device__ __forceinline__ void fq_scan16(const uint8_t* in, uint64_t o, uint64_t lim, uint64_t base, uint32_t& c, long long l[4]) {
  if(o >= lim) return;
  uint8_t b[16];
  if(o + 16 <= lim) {
    *reinterpret_cast<uint4*>(b) = __ldg(reinterpret_cast<const uint4*>(in + o));
  } else {
#pragma unroll
    for(int i = 0; i < 16; ++i) b[i] = o + i < lim ? in[o + i] : 0;
  }
#pragma unroll
  for(int i = 0; i < 16; ++i) {
    if(b[i] == '\n') {
      ++c;
      const long long pos = (long long)(o + i - base);
      const uint32_t r = c & 3u;
      l[0] = r == 0 ? pos : l[0]; l[1] = r == 1 ? pos : l[1]; l[2] = r == 2 ? pos : l[2]; l[3] = r == 3 ? pos : l[3];
    }
  }
}

// One CTA of 256 threads per tile, 64 bytes a thread.
__global__ void __launch_bounds__(256) fastq_tiles_kernel(const uint8_t* in, uint64_t n, FqTile* tiles) {
  __shared__ uint32_t sm_sum[33];
  __shared__ long long sm_max[4 * 32];
  const uint64_t t0 = (uint64_t)blockIdx.x * FQ_TILE, my = t0 + (uint64_t)threadIdx.x * 64;
  uint32_t c = 0;
  long long l[4] = {-1, -1, -1, -1};
#pragma unroll
  for(int j = 0; j < 4; ++j) fq_scan16(in, my + 16 * j, n, t0, c, l);
  uint32_t total = 0;
  const uint32_t pre = block_excl_sum(c, sm_sum, &total);
  // the thread's newline of local index i has tile index pre + i: tile residue s is local residue s - pre
  long long v[4];
  for(int s = 0; s < 4; ++s) v[s] = l[(s - pre) & 3u];
  block_max4(v, sm_max);
  if(threadIdx.x == 0) {
    FqTile t;
    t.n = total;
    for(int s = 0; s < 4; ++s) t.last[s] = (int32_t)v[s];
    tiles[blockIdx.x] = t;
  }
}

// One CTA of 1024 threads: the line phase at every tile start, the last record end up to every tile, then the cuts one
// after the other (each rescans the head of one tile, FQ_TILE / 1024 = 16 bytes a thread).
__global__ void __launch_bounds__(1024) fastq_resolve_kernel(const uint8_t* in, uint64_t n, uint32_t lines_mod4, uint64_t target,
                                                             uint64_t cap, const FqTile* tiles, uint64_t n_tiles, uint8_t* phase,
                                                             unsigned long long* through, FqResult* res, unsigned long long* cuts) {
  __shared__ uint32_t sm_sum[33];
  __shared__ long long sm_max[4 * 32];
  const uint64_t per = (n_tiles + blockDim.x - 1) / blockDim.x;
  const uint64_t a = min(n_tiles, per * threadIdx.x), b = min(n_tiles, a + per);
  // phases: an exclusive sum of the newline counts (mod 4) over the tiles
  uint32_t mine = 0;
  for(uint64_t t = a; t < b; ++t) mine += tiles[t].n & 3u;
  uint32_t total = 0;
  uint32_t ph = lines_mod4 + block_excl_sum(mine, sm_sum, &total);
  long long m = 0;                          // last record end (offset behind its '\n'; 0: none) in this thread's tiles
  for(uint64_t t = a; t < b; ++t) {
    phase[t] = (uint8_t)(ph & 3u);
    const int32_t e = tiles[t].last[(4u - (ph & 3u)) & 3u];     // tile index i ends a record when phase + i = 0 (mod 4)
    if(e >= 0) m = (long long)(t * FQ_TILE) + e + 1;
    through[t] = (unsigned long long)m;     // (this thread's part of the running maximum; completed below)
    ph += tiles[t].n & 3u;
  }
  // the rest of the running maximum: the ends grow with the thread, so the last thread in front that has one gives it
  __shared__ long long sm_last[1024];
  sm_last[threadIdx.x] = m;
  __syncthreads();
  long long before = 0;
  for(int i = (int)threadIdx.x - 1; i >= 0 && !before; --i) before = sm_last[i];
  for(uint64_t t = a; t < b && !through[t]; ++t) through[t] = (unsigned long long)before;
  __syncthreads();
  // the cuts, one after the other
  unsigned long long count = 0, status = 0, fail_at = 0;
  uint64_t o = 0;
  while(o + target < n) {
    const uint64_t lim = o + target, t = (lim - 1) / FQ_TILE, t0 = t * FQ_TILE;
    uint32_t c = 0;
    long long l[4] = {-1, -1, -1, -1};
    fq_scan16(in, t0 + (uint64_t)threadIdx.x * 16, lim, t0, c, l);
    uint32_t tot = 0;
    const uint32_t pre = block_excl_sum(c, sm_sum, &tot);
    const uint32_t want = (4u - phase[t]) & 3u;
    long long w[4] = {l[(want - pre) & 3u], -1, -1, -1};
    block_max4(w, sm_max);
    const uint64_t e = w[0] >= 0 ? t0 + (uint64_t)w[0] + 1 : (t ? (uint64_t)through[t - 1] : 0);
    if(e <= o) { status = 1; fail_at = o; break; }
    if(count >= cap) { status = 2; fail_at = o; break; }
    if(threadIdx.x == 0) cuts[count] = e;
    ++count;
    o = e;
  }
  if(threadIdx.x == 0) {
    res->n_cuts = count; res->end_lines = (lines_mod4 + total) & 3u; res->status = status; res->fail_at = fail_at;
  }
}

}  // namespace

size_t fastq_cuts_scratch(size_t n, size_t cap) {
  const size_t tiles = (n + FQ_TILE - 1) / FQ_TILE + 1;
  return sizeof(FqResult) + cap * 8 + tiles * (sizeof(FqTile) + 8 + 1) + 64;
}

int fastq_cuts(const uint8_t* in, size_t n, uint32_t lines_mod4, uint64_t target, size_t cap, void* scratch, cudaStream_t st) {
  const uint64_t n_tiles = (n + FQ_TILE - 1) / FQ_TILE;
  uint8_t* p = (uint8_t*)scratch;
  FqResult* res = (FqResult*)p;
  unsigned long long* cuts = (unsigned long long*)(p + sizeof(FqResult));
  unsigned long long* through = cuts + cap;
  FqTile* tiles = (FqTile*)(through + n_tiles + 1);
  uint8_t* phase = (uint8_t*)(tiles + n_tiles + 1);
  int launches = 0;
  if(n_tiles) { fastq_tiles_kernel<<<(unsigned)n_tiles, 256, 0, st>>>(in, n, tiles); ++launches; }
  fastq_resolve_kernel<<<1, 1024, 0, st>>>(in, n, lines_mod4 & 3u, target, cap, tiles, n_tiles, phase, through, res, cuts);
  return launches + 1;
}

int count_newlines(const uint8_t* in, size_t n, unsigned long long* count, int n_sm, cudaStream_t st) {
  if(n == 0) return 0;
  const uint64_t vecs = n / 16 + 1;
  const int grid = (int)(vecs / 256 + 1 < (uint64_t)n_sm * 8 ? vecs / 256 + 1 : (uint64_t)n_sm * 8);
  count_newlines_kernel<<<grid, 256, 0, st>>>(in, n, count);
  return 1;
}

}  // namespace jfnl
