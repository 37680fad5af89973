// jf_newline.cu -- the newline count of jf_newline.cuh: 16-byte loads, four SWAR byte compares per load.
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

}  // namespace

int count_newlines(const uint8_t* in, size_t n, unsigned long long* count, int n_sm, cudaStream_t st) {
  if(n == 0) return 0;
  const uint64_t vecs = n / 16 + 1;
  const int grid = (int)(vecs / 256 + 1 < (uint64_t)n_sm * 8 ? vecs / 256 + 1 : (uint64_t)n_sm * 8);
  count_newlines_kernel<<<grid, 256, 0, st>>>(in, n, count);
  return 1;
}

}  // namespace jfnl
