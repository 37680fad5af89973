// Shared-memory atomic throughput (what K1's slot reservation, the window scatter and the window insert are made of).
//   1. random addresses over tables of several sizes: returning add, non-returning add, CAS, plain load+store, load;
//   2. the lane patterns of one warp instruction: all 32 lanes on 1 address, on 32 distinct banks (lane i -> word i), on
//      32 random words of 1024 (K1's atomicAdd on a region's ring counter, 1024 regions) and of 2048 (K1's hash table
//      loads, one 11-bit table), for returning add, plain store and load.
// Figures: operations (lanes) per clock per SM at the SM clock the card reports, and warp instructions per clock per SM.
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>
__device__ __forceinline__ uint32_t mix(uint32_t x) { x ^= x >> 16; x *= 0x7feb352dU; x ^= x >> 15; x *= 0x846ca68bU; x ^= x >> 16; return x; }
template<int MODE>
__global__ void __launch_bounds__(1024, 1) k(uint32_t nb_mask, uint32_t iters, uint32_t* out) {
  extern __shared__ uint32_t sm[];
  for(uint32_t i = threadIdx.x; i <= nb_mask; i += blockDim.x) sm[i] = 0;
  __syncthreads();
  uint32_t x = mix(blockIdx.x * 1024u + threadIdx.x + 1u), acc = 0;
  for(uint32_t it = 0; it < iters; ++it) {
#pragma unroll
    for(int u = 0; u < 4; ++u) {
      x = x * 1664525u + 1013904223u;
      const uint32_t a = (x >> 8) & nb_mask;
      if(MODE == 0) acc += atomicAdd(&sm[a], 1u);                 // returning
      else if(MODE == 1) atomicAdd(&sm[a], 1u);                   // result unused
      else if(MODE == 2) acc += atomicCAS(&sm[a], 0u, x | 1u);     // CAS
      else if(MODE == 3) { uint32_t v = sm[a]; sm[a] = v + 1; acc += v; }   // plain load + store (racy on purpose)
      else { acc += sm[a]; }                                      // plain load
    }
  }
  __syncthreads();
  if(acc == 0x12345678u || sm[threadIdx.x & nb_mask] == 0xFFFFFFFFu) out[0] = acc;
}
// lane patterns: PAT 0 = every lane on word 0, 1 = lane i on word i, 2 = random words of nb (mask nb_mask)
// OP 0 = returning atomicAdd, 1 = plain store, 2 = plain load
template<int PAT, int OP>
__global__ void __launch_bounds__(1024, 1) kp(uint32_t nb_mask, uint32_t iters, uint32_t* out) {
  extern __shared__ uint32_t sm[];
  for(uint32_t i = threadIdx.x; i <= nb_mask; i += blockDim.x) sm[i] = 0;
  __syncthreads();
  const uint32_t lane = threadIdx.x & 31u;
  uint32_t x = mix(blockIdx.x * 1024u + threadIdx.x + 1u), acc = 0;
  for(uint32_t it = 0; it < iters; ++it) {
#pragma unroll
    for(int u = 0; u < 4; ++u) {
      x = x * 1664525u + 1013904223u;
      const uint32_t a = PAT == 0 ? 0u : PAT == 1 ? lane : ((x >> 8) & nb_mask);
      if(OP == 0) acc += atomicAdd(&sm[a], 1u);
      else if(OP == 1) reinterpret_cast<volatile uint32_t*>(sm)[a] = x;   // (volatile: every store is issued)
      else acc += sm[a ^ (acc & 1u)];            // (the load feeds the next address: no hoisting)
    }
  }
  __syncthreads();
  if(acc == 0x12345678u || sm[threadIdx.x & nb_mask] == 0xFFFFFFFFu) out[0] = acc;
}
static double g_ghz = 1.98;
static int g_sms = 132;
template<typename K> double time_it(K kern, uint32_t nb, uint32_t* d) {
  cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
  cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
  const uint32_t iters = 4096;
  kern<<<g_sms, 1024, nb * 4, 0>>>(nb - 1, 64, d);
  cudaEventRecord(a);
  kern<<<g_sms, 1024, nb * 4, 0>>>(nb - 1, iters, d);
  cudaEventRecord(b); cudaEventSynchronize(b);
  float ms; cudaEventElapsedTime(&ms, a, b);
  cudaEventDestroy(a); cudaEventDestroy(b);
  return (double)g_sms * 1024 * iters * 4 / ms / 1e6;      // G lane-operations per second
}
template<int MODE> void run(const char* name, uint32_t nb, uint32_t* d) {
  const double g = time_it(k<MODE>, nb, d);
  printf("%-22s bins %6u : %7.2f G ops/s  = %5.2f ops/clk/SM  [%s]\n", name, nb, g, g / g_sms / g_ghz, cudaGetErrorString(cudaGetLastError()));
}
template<int PAT, int OP> void runp(const char* op, const char* pat, uint32_t nb, uint32_t* d) {
  const double g = time_it(kp<PAT, OP>, nb, d);
  printf("%-10s %-24s : %7.2f G lanes/s = %6.2f lanes/clk/SM = %5.3f warp instr/clk/SM  [%s]\n", op, pat, g, g / g_sms / g_ghz,
         g / g_sms / g_ghz / 32, cudaGetErrorString(cudaGetLastError()));
}
int main() {
  cudaDeviceProp prop; cudaGetDeviceProperties(&prop, 0);
  int clk_khz = 0; cudaDeviceGetAttribute(&clk_khz, cudaDevAttrClockRate, 0);
  g_ghz = clk_khz / 1e6; g_sms = prop.multiProcessorCount;
  printf("%s, %d SMs, SM clock %.3f GHz (per-clock figures assume it)\n", prop.name, g_sms, g_ghz);
  uint32_t* d; cudaMalloc(&d, 64);
  for(uint32_t nb : {512u, 2048u, 16384u}) {
    run<0>("atomicAdd returning", nb, d); run<1>("atomicAdd no result", nb, d); run<2>("atomicCAS", nb, d);
    run<3>("load+store", nb, d); run<4>("load", nb, d);
  }
  runp<0, 0>("atomicAdd", "1 address", 1024, d);
  runp<1, 0>("atomicAdd", "32 distinct banks", 1024, d);
  runp<2, 0>("atomicAdd", "32 random of 1024", 1024, d);
  runp<2, 0>("atomicAdd", "32 random of 2048", 2048, d);
  runp<0, 1>("store", "1 address", 1024, d);
  runp<1, 1>("store", "32 distinct banks", 1024, d);
  runp<2, 1>("store", "32 random of 1024", 1024, d);
  runp<1, 2>("load", "32 distinct banks", 1024, d);
  runp<2, 2>("load", "32 random of 1024", 1024, d);
  runp<2, 2>("load", "32 random of 2048", 2048, d);
  return 0;
}
