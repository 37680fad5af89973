// jf_bloom.cu -- instantiations of the kernels of sharded Bloom counting (jf_bloom.cuh).
// The kernel headers are compiled here under a namespace of their own, as in jf_wide.cu.
#include <cuda_runtime.h>
#define jfk jfk_bloom
#include "jf_kernels.cuh"
#undef jfk
#include "jf_bloom.cuh"

namespace jfk_bloom {

// Fold another Bloom counter into words [0, n) of `dst` (bloom_counter2.hpp:56-107; the two-bit form of bloom_count,
// jf_device.cuh).  Every position is (hit, hit again): after both counters' hits it is hit = hit_a | hit_b,
// again = again_a | again_b | (hit_a & hit_b) -- min(2, hits_a + hits_b), whatever the order of the hits.
__global__ void __launch_bounds__(256) bloom_fold_kernel(uint32_t* __restrict__ dst, const uint32_t* __restrict__ src, uint64_t n) {
  for(uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
    const uint32_t a = dst[i], b = __ldg(&src[i]);
    dst[i] = a | b | ((a & b & 0x55555555u) << 1);
  }
}

}  // namespace jfk_bloom

namespace jfbl {
using namespace jfk_bloom;

const Kernels& kernels() {
  static const Kernels k = {
    { (const void*)insert_keys_bf_kernel<1, 32>, (const void*)insert_keys_bf_kernel<1, 64>, (const void*)insert_keys_bf_kernel<1, 128>,
      (const void*)insert_keys_bf_kernel<2, 64>, (const void*)insert_keys_bf_kernel<2, 128> },
    { (const void*)stage_keys_bf_kernel<1>, (const void*)stage_keys_bf_kernel<2> },
    (const void*)bloom_fold_kernel,
  };
  return k;
}

}  // namespace jfbl
