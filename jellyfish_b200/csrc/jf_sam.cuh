// jf_sam.cuh -- SAM and BAM input: kernels that rewrite a batch of SAM lines or BAM records in device memory as 4-line
// FASTQ records "@\n SEQ \n+\n QUAL \n", which the extraction kernels then count as they count FASTQ.
//
// The reference reads alignment files through htslib and hands each record's SEQ and qualities to the same code as a FASTQ
// read (mer_overlap_sequence_parser.hpp:220-253, whole_sequence_parser.hpp:192-208): bases decoded by sam_format.hpp
// (A, C, G, T, anything else N), the quality character phred + '!', FLAG ignored.  A FASTQ record per alignment record gives
// exactly that, the N between reads, the k-1 seam, -Q, the Bloom filters and k > 64 included.
//
// The kernels are compiled in a translation unit of their own, jf_sam.cu, and started through the host functions below: the
// engine's module keeps exactly the kernels it had (split compilation assigns functions to partitions over the whole module).
#ifndef JF_SAM_CUH
#define JF_SAM_CUH
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

namespace jfsam {

enum : uint32_t {                  // what is wrong with the first malformed record of a batch (Result::err & 3)
  ERR_FIELDS = 1,                  // a SAM line with fewer than 11 tab-separated fields
  ERR_QUAL_LEN = 2,                // SEQ and QUAL of different lengths (QUAL not '*')
  ERR_BAM_RECORD = 3,              // a BAM record whose name, CIGAR, SEQ and QUAL run past its block_size
};

struct Result {                    // written by the kernels, read back by the host after each batch
  unsigned long long n_recs;       // candidate records (SAM: lines that are neither headers nor blank)
  unsigned long long out_bytes;    // bytes of FASTQ written
  unsigned long long consumed;     // SAM: input bytes up to and including the last newline (all of them for a final batch)
  unsigned long long last_nl;      // SAM: 1 + position of the last newline (0: none)
  unsigned long long err;          // ~0 = none; else (byte offset of the first bad record << 2) | ERR_*
};

// Device scratch of a batch of at most `in_cap` input bytes (in_cap <= 2^30).  The FASTQ output needs at most 2 * in_cap bytes.
size_t scratch_bytes(size_t in_cap);
// The largest number of BAM records a batch of `in_cap` bytes holds (each record has at least 36 bytes).
inline size_t max_bam_records(size_t in_cap) { return in_cap / 36 + 1; }

// Transcode the SAM text [in, in + n) (any alignment; it starts at a line start).  Lines that end inside the batch are
// transcoded, and with `final` the last line without a newline too.  Header lines ('@') and blank lines are skipped.  Returns
// the number of kernels launched.  `res` (device memory) receives the Result.
int sam_transcode(const uint8_t* in, size_t n, bool final, uint8_t* out, void* scratch, size_t in_cap, Result* res, cudaStream_t st);
// Transcode the n_recs BAM records at byte offsets offs[0..n_recs) of [in, in + n) (offs: device memory; the host has walked
// the block_size chain, so every record lies inside the batch).
int bam_transcode(const uint8_t* in, size_t n, const uint32_t* offs, uint32_t n_recs, uint8_t* out, void* scratch, size_t in_cap,
                  Result* res, cudaStream_t st);

}  // namespace jfsam
#endif
