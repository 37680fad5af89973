// jf_newline.cuh -- count the '\n' bytes of a device range (jfgpu_count_newlines).  The line index at which a share of a
// FASTQ file starts is the number of newlines in front of it; every rank tallies the newlines of its own share while it
// counts it, and the ranks compare the tallies to check that every share starts on a 4-line record.
//
// Compiled in a translation unit of its own, jf_newline.cu, so that the engine's module keeps exactly the kernels it had.
#ifndef JF_NEWLINE_CUH
#define JF_NEWLINE_CUH
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

namespace jfnl {

// Add the '\n' bytes of [in, in + n) (any alignment) to *count (device memory).  Returns the number of kernels launched.
int count_newlines(const uint8_t* in, size_t n, unsigned long long* count, int n_sm, cudaStream_t st);

}  // namespace jfnl
#endif
