// jf_newline.cuh -- count the '\n' bytes of a device range (jfgpu_count_newlines), and cut FASTQ text behind whole records
// (jfgpu_fastq_cuts).  The line index at which a share of a
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

// Record-aligned cuts of FASTQ text (jfgpu_fastq_cuts).  A record ends behind a '\n' in front of which the number of lines,
// counted from lines_mod4 at `in`, is a multiple of 4.  Cut c_0 = 0; c_i is the last record end <= c_{i-1} + target, for as
// long as c_{i-1} + target < n, so that every piece [c_{i-1}, c_i) and the last one [c_m, n) holds at most `target` bytes.
// FQ_TILE-byte tiles: one kernel reads every byte once (per tile: newlines, and the last newline of each residue of its
// index), one CTA resolves the cuts, rescanning at most one tile's head per cut.  `in` is 16-byte aligned.
constexpr uint32_t FQ_TILE = 16384;

// What the resolving CTA leaves in the first words of the scratch: the number of cuts, the lines (mod 4) at the end of the
// text, and on failure 1 (no record end within target bytes of piece start `fail_at`) or 2 (more cuts than `cap`).
struct FqResult { unsigned long long n_cuts, end_lines, status, fail_at; };

// Bytes of device scratch for a text of n bytes and at most `cap` cuts.
size_t fastq_cuts_scratch(size_t n, size_t cap);
// Launch both kernels on st; the result (FqResult) and then the cuts (uint64 each) are at the start of `scratch`.  Returns
// the number of kernels launched.
int fastq_cuts(const uint8_t* in, size_t n, uint32_t lines_mod4, uint64_t target, size_t cap, void* scratch, cudaStream_t st);

}  // namespace jfnl
#endif
