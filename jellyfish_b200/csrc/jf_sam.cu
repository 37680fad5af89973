// jf_sam.cu -- SAM and BAM records rewritten as 4-line FASTQ in device memory (jf_sam.cuh).
//
// SAM, per batch: (1) every tile counts the lines that start in it and are neither headers ('@') nor blank, (2) one block
// scans the tile counts, (3) every tile writes the start offsets of its lines in order, (4) one warp per line finds the tabs
// that bound SEQ (field 10) and QUAL (field 11) with ballots over 32-byte strides and checks the field count and lengths.
// BAM: the host gives the record offsets; (4') one thread per record reads its fixed fields.  Both then (5, 6) scan the
// output lengths, 2 * len + 6 per record, and (7) one warp per record writes "@\n SEQ \n+\n QUAL \n" at its offset, one byte
// per lane.
//
// Positions are offsets from the 16-byte aligned address at or below `in`: the input [lo, hi) is read with aligned 16-byte
// loads (a batch of a device feed may start anywhere).
#include "jf_sam.cuh"

namespace jfsam {
namespace {

constexpr int TILE_THREADS = 256;
constexpr int TILE_WORDS = 4;                                    // 16-byte words per thread and tile
constexpr uint32_t TILE_BYTES = TILE_THREADS * TILE_WORDS * 16;  // 16 KB
constexpr int SCAN_BLOCKS = 1024;                                // blocks of the record scan (a fixed grid: the record count stays on the device)

struct Scratch {
  uint32_t* tile_cnt;              // per tile: its record lines, then their first index
  uint32_t* starts;                // SAM: offset of every record line
  uint32_t* seq;                   // offset of SEQ
  uint32_t* qual;                  // offset of QUAL, NO_QUAL for '*'
  uint32_t* len;                   // bases (0: nothing to write)
  uint32_t* ooff;                  // output offset inside the record's scan block
  uint32_t* boff;                  // SCAN_BLOCKS: output offset of every scan block
  size_t rec_cap;
};
constexpr uint32_t NO_QUAL = 0xffffffffu;

// Every line of at least 11 fields has 10 tabs and a line end: a batch of n bytes holds at most n / 11 + 1 such lines.  More
// line starts than that mean a line with fewer fields.
size_t rec_capacity(size_t in_cap) { return in_cap / 11 + 2; }
size_t n_tiles_for(size_t hi) { return (hi + TILE_BYTES - 1) / TILE_BYTES; }

Scratch carve(void* p, size_t in_cap) {
  Scratch s;
  s.rec_cap = rec_capacity(in_cap);
  const size_t tiles = n_tiles_for(in_cap + 16) + 1;
  uint32_t* q = (uint32_t*)p;
  s.tile_cnt = q; q += tiles;
  s.starts = q; q += s.rec_cap;
  s.seq = q; q += s.rec_cap;
  s.qual = q; q += s.rec_cap;
  s.len = q; q += s.rec_cap;
  s.ooff = q; q += s.rec_cap;
  s.boff = q;
  return s;
}

__device__ __forceinline__ void set_error(Result* res, uint64_t pos, uint32_t code) {
  atomicMax(&res->err, ~((unsigned long long)pos << 2 | code));    // the first bad record in the batch wins
}

// exclusive prefix sum over the block; *total = the block's sum.  `sm` holds 32 words.
template<int NT>
__device__ uint32_t block_excl_scan(uint32_t v, uint32_t* total, uint32_t* sm) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  uint32_t x = v;
#pragma unroll
  for(int d = 1; d < 32; d <<= 1) { const uint32_t y = __shfl_up_sync(0xffffffffu, x, d); if(lane >= d) x += y; }
  if(lane == 31) sm[warp] = x;
  __syncthreads();
  if(warp == 0) {
    uint32_t y = lane < NT / 32 ? sm[lane] : 0;
#pragma unroll
    for(int d = 1; d < 32; d <<= 1) { const uint32_t z = __shfl_up_sync(0xffffffffu, y, d); if(lane >= d) y += z; }
    sm[lane] = y;
  }
  __syncthreads();
  const uint32_t pre = warp ? sm[warp - 1] : 0;
  *total = sm[NT / 32 - 1];
  __syncthreads();
  return pre + x - v;
}

// bit 8j+7 set for every byte j of x equal to c
__device__ __forceinline__ uint32_t bytes_equal(uint32_t x, uint32_t c4) {
  const uint32_t t = x ^ c4;
  return ~(((t & 0x7f7f7f7fu) + 0x7f7f7f7fu) | t | 0x7f7f7f7fu);
}

// Does a record line start at s?  Not past the data, not a header line, not blank ("\n" or "\r\n").
__device__ __forceinline__ bool record_start(const uint8_t* A, uint32_t s, uint32_t hi) {
  if(s >= hi) return false;
  const uint8_t c = A[s];
  if(c == '@' || c == '\n') return false;
  return !(c == '\r' && s + 1 < hi && A[s + 1] == '\n');
}

// The record-line starts of 16-byte word w, in order: the batch's own start (lo), then the byte behind every newline.  Calls
// f(s) for each; returns 1 + the position of the word's last newline (0: none).
template<typename F>
__device__ __forceinline__ uint32_t word_starts(const uint8_t* A, uint32_t w, uint32_t lo, uint32_t hi, F&& f) {
  const uint32_t base = w * 16;
  if(base >= hi) return 0;
  if(base <= lo && lo < base + 16 && record_start(A, lo, hi)) f(lo);
  const uint4 v = *reinterpret_cast<const uint4*>(A + base);
  const uint32_t x[4] = { v.x, v.y, v.z, v.w };
  uint32_t last = 0;
#pragma unroll
  for(int i = 0; i < 4; ++i) {
    uint32_t m = bytes_equal(x[i], 0x0a0a0a0au);
    while(m) {
      const uint32_t q = base + 4 * i + ((__ffs(m) - 1) >> 3);
      m &= m - 1;
      if(q < lo || q >= hi) continue;
      last = q + 1;
      if(record_start(A, q + 1, hi)) f(q + 1);
    }
  }
  return last;
}

// (1) record lines per tile; the last newline of the batch
__global__ void __launch_bounds__(TILE_THREADS) sam_count_kernel(const uint8_t* A, uint32_t lo, uint32_t hi, uint32_t* tile_cnt, Result* res) {
  __shared__ uint32_t sm[32];
  uint32_t c = 0, last = 0;
  for(int it = 0; it < TILE_WORDS; ++it) {
    const uint32_t w = (blockIdx.x * TILE_WORDS + it) * TILE_THREADS + threadIdx.x;
    last = max(last, word_starts(A, w, lo, hi, [&](uint32_t) { ++c; }));
  }
  uint32_t total;
  block_excl_scan<TILE_THREADS>(c, &total, sm);
  if(threadIdx.x == 0) tile_cnt[blockIdx.x] = total;
  if(last) atomicMax(&res->last_nl, (unsigned long long)last);
}

// (2) first record index of every tile; the number of records and the bytes the batch consumes
__global__ void __launch_bounds__(1024) sam_tiles_kernel(uint32_t* tile_cnt, uint32_t n_tiles, uint32_t rec_cap, uint32_t lo, uint32_t hi,
                                                         uint32_t final, Result* res) {
  __shared__ uint32_t sm[32];
  uint32_t run = 0;
  for(uint32_t b = 0; b < n_tiles; b += 1024) {
    const uint32_t i = b + threadIdx.x;
    const uint32_t v = i < n_tiles ? tile_cnt[i] : 0;
    uint32_t total;
    const uint32_t x = block_excl_scan<1024>(v, &total, sm);
    if(i < n_tiles) tile_cnt[i] = run + x;
    run += total;
  }
  if(threadIdx.x == 0) {
    // More line starts than rec_cap: one of the first rec_cap - 1 lines is shorter than 11 bytes (rec_capacity), and (4) reports
    // the first such line.  The error here only backstops that, at a position no line start reaches, so it never wins.
    res->n_recs = min(run, rec_cap);
    if(run > rec_cap) set_error(res, hi - lo, ERR_FIELDS);
    const unsigned long long nl = res->last_nl;
    res->consumed = final ? hi - lo : nl ? nl - lo : 0;
  }
}

// (3) the start of every record line, in input order
__global__ void __launch_bounds__(TILE_THREADS) sam_index_kernel(const uint8_t* A, uint32_t lo, uint32_t hi, const uint32_t* tile_first,
                                                                 uint32_t* starts, uint32_t rec_cap) {
  __shared__ uint32_t sm[32];
  uint32_t next = tile_first[blockIdx.x];
  for(int it = 0; it < TILE_WORDS; ++it) {
    const uint32_t w = (blockIdx.x * TILE_WORDS + it) * TILE_THREADS + threadIdx.x;
    uint32_t c = 0;
    word_starts(A, w, lo, hi, [&](uint32_t) { ++c; });
    uint32_t total;
    uint32_t i = next + block_excl_scan<TILE_THREADS>(c, &total, sm);
    if(c) word_starts(A, w, lo, hi, [&](uint32_t s) { if(i < rec_cap) starts[i] = s; ++i; });
    next += total;
  }
}

// (4) one warp per record line: SEQ and QUAL
__global__ void __launch_bounds__(256) sam_parse_kernel(const uint8_t* A, uint32_t lo, uint32_t hi, uint32_t final, const uint32_t* starts,
                                                        Result* res, uint32_t* seq, uint32_t* qual, uint32_t* len) {
  const uint32_t lane = threadIdx.x & 31;
  const uint64_t n_recs = res->n_recs;
  const uint64_t end_ok = lo + res->consumed;       // lines that start at or behind it end in the next batch
  for(uint64_t r = (blockIdx.x * (uint64_t)blockDim.x + threadIdx.x) / 32; r < n_recs; r += gridDim.x * (uint64_t)blockDim.x / 32) {
    const uint32_t s = starts[r];
    uint32_t t9 = 0, t10 = 0, qend = 0, tabs = 0;
    if(s >= end_ok && !final) { if(lane == 0) len[r] = 0; continue; }
    for(uint32_t p = s; ; p += 32) {
      const uint32_t q = p + lane;
      const uint8_t c = q < hi ? A[q] : 0;
      const uint32_t valid = __ballot_sync(0xffffffffu, q < hi);
      uint32_t tm = __ballot_sync(0xffffffffu, c == '\t');
      const uint32_t nm = __ballot_sync(0xffffffffu, c == '\n');
      if(nm) tm &= (nm & (0u - nm)) - 1;           // tabs in front of the line's newline
      while(tm && tabs < 11) {
        const uint32_t at = p + __ffs(tm) - 1;
        tm &= tm - 1;
        ++tabs;
        if(tabs == 9) t9 = at; else if(tabs == 10) t10 = at; else if(tabs == 11) qend = at;
      }
      if(tabs == 11) break;
      if(nm || valid != 0xffffffffu) {
        // the line ends at its newline (one '\r' in front of it goes with it) or at the end of the data
        qend = nm ? p + __ffs(nm) - 1 : hi;
        if(nm && tabs == 10 && qend > t10 + 1 && A[qend - 1] == '\r') --qend;
        break;
      }
    }
    if(lane != 0) continue;
    if(tabs < 10) { set_error(res, s - lo, ERR_FIELDS); len[r] = 0; continue; }
    uint32_t sl = t10 - t9 - 1, ql = qend - t10 - 1;
    if(sl == 1 && A[t9 + 1] == '*') sl = 0;
    const bool no_qual = ql == 1 && A[t10 + 1] == '*';
    if(!no_qual && ql != sl) { set_error(res, s - lo, ERR_QUAL_LEN); len[r] = 0; continue; }
    seq[r] = t9 + 1; qual[r] = no_qual ? NO_QUAL : t10 + 1; len[r] = sl;
  }
}

// (4') one thread per BAM record (SAM specification 4.2): block_size, refID, pos, l_read_name, mapq, bin, n_cigar_op, flag, l_seq,
// next_refID, next_pos, tlen, read_name, cigar, seq (4-bit codes, two per byte), qual (phred), tags
__device__ __forceinline__ uint32_t le32(const uint8_t* p) { return p[0] | (uint32_t)p[1] << 8 | (uint32_t)p[2] << 16 | (uint32_t)p[3] << 24; }
__global__ void __launch_bounds__(256) bam_parse_kernel(const uint8_t* A, uint32_t lo, const uint32_t* offs, uint32_t n_recs, Result* res,
                                                        uint32_t* seq, uint32_t* qual, uint32_t* len) {
  const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
  if(r == 0) res->n_recs = n_recs;
  if(r >= n_recs) return;
  const uint32_t b = lo + offs[r];
  const uint8_t* p = A + b;
  const uint64_t block = le32(p), l_name = p[12], n_cigar = p[16] | (uint32_t)p[17] << 8;
  const int32_t l_seq = (int32_t)le32(p + 20);
  const uint64_t s = 36 + l_name + 4 * n_cigar, q = s + ((uint64_t)l_seq + 1) / 2;
  if(l_seq < 0 || q + (uint64_t)l_seq > 4 + block) { set_error(res, offs[r], ERR_BAM_RECORD); len[r] = 0; return; }
  seq[r] = b + (uint32_t)s; qual[r] = b + (uint32_t)q; len[r] = (uint32_t)l_seq;
}

__device__ __forceinline__ uint32_t out_len(uint32_t l) { return l ? 2 * l + 6 : 0; }

// (5) output offsets inside each of SCAN_BLOCKS contiguous ranges of records
__global__ void __launch_bounds__(256) scan_local_kernel(const uint32_t* len, const Result* res, uint32_t* ooff, uint32_t* boff) {
  __shared__ uint32_t sm[32];
  const uint64_t n = res->n_recs, per = (n + gridDim.x - 1) / gridDim.x;
  const uint64_t b0 = blockIdx.x * per, b1 = min(n, b0 + per);
  uint32_t run = 0;
  for(uint64_t b = b0; b < b1; b += 256) {
    const uint64_t i = b + threadIdx.x;
    const uint32_t v = i < b1 ? out_len(len[i]) : 0;
    uint32_t total;
    const uint32_t x = block_excl_scan<256>(v, &total, sm);
    if(i < b1) ooff[i] = run + x;
    run += total;
  }
  if(threadIdx.x == 0) boff[blockIdx.x] = run;
}

// (6) offsets of the ranges; the batch's output size
__global__ void __launch_bounds__(SCAN_BLOCKS) scan_blocks_kernel(uint32_t* boff, Result* res) {
  __shared__ uint32_t sm[32];
  uint32_t total;
  const uint32_t x = block_excl_scan<SCAN_BLOCKS>(boff[threadIdx.x], &total, sm);
  boff[threadIdx.x] = x;
  if(threadIdx.x == 0) res->out_bytes = total;
}

// (7) one warp per record: "@\n" SEQ "\n+\n" QUAL "\n"
template<bool BAM>
__global__ void __launch_bounds__(256) emit_kernel(const uint8_t* A, const Result* res, const uint32_t* seq, const uint32_t* qual,
                                                   const uint32_t* len, const uint32_t* ooff, const uint32_t* boff, uint8_t* out) {
  const uint32_t lane = threadIdx.x & 31;
  const uint64_t n = res->n_recs, per = (n + SCAN_BLOCKS - 1) / SCAN_BLOCKS;
  for(uint64_t r = (blockIdx.x * (uint64_t)blockDim.x + threadIdx.x) / 32; r < n; r += gridDim.x * (uint64_t)blockDim.x / 32) {
    const uint32_t l = len[r];
    if(!l) continue;
    uint8_t* o = out + boff[r / per] + ooff[r];
    const uint32_t sp = seq[r], qp = qual[r];
    for(uint32_t i = lane; i < 2 * l + 6; i += 32) {
      uint8_t c;
      if(i < 2) c = i ? '\n' : '@';
      else if(i < 2 + l) {
        const uint32_t j = i - 2;
        if(BAM) {
          const uint8_t b = A[sp + j / 2];
          const uint32_t code = j & 1 ? b & 15 : b >> 4;            // sam_format.hpp: 1 A, 2 C, 4 G, 8 T, anything else N
          c = code == 1 ? 'A' : code == 2 ? 'C' : code == 4 ? 'G' : code == 8 ? 'T' : 'N';
        } else {
          c = A[sp + j];
          const uint8_t u = c & 0xdf;                               // ACGT in either case are bases, any other byte an N
          if(u != 'A' && u != 'C' && u != 'G' && u != 'T') c = 'N';
        }
      } else if(i < 5 + l) c = i == 3 + l ? '+' : '\n';
      else if(i < 5 + 2 * l) {
        const uint32_t j = i - 5 - l;
        // BAM: phred + '!' (mod 256: a missing QUAL, 0xff, becomes 0x20); SAM: the character itself, 0x20 for '*' (htslib
        // stores '*' as 0xff, whole_sequence_parser.hpp:192-208 adds '!')
        c = BAM ? (uint8_t)(A[qp + j] + 33) : qp == NO_QUAL ? (uint8_t)0x20 : A[qp + j];
      } else c = '\n';
      o[i] = c;
    }
  }
}

int record_grid() {
  static int g = 0;
  if(!g) {
    int dev = 0, sms = 132;
    if(cudaGetDevice(&dev) == cudaSuccess) cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    g = sms * 8;
  }
  return g;
}

// (5)-(7): 3 launches
int scan_and_emit(const uint8_t* A, bool bam, const Scratch& s, uint8_t* out, Result* res, cudaStream_t st) {
  scan_local_kernel<<<SCAN_BLOCKS, 256, 0, st>>>(s.len, res, s.ooff, s.boff);
  scan_blocks_kernel<<<1, SCAN_BLOCKS, 0, st>>>(s.boff, res);
  if(bam) emit_kernel<true><<<record_grid(), 256, 0, st>>>(A, res, s.seq, s.qual, s.len, s.ooff, s.boff, out);
  else emit_kernel<false><<<record_grid(), 256, 0, st>>>(A, res, s.seq, s.qual, s.len, s.ooff, s.boff, out);
  return 3;
}

}  // namespace

size_t scratch_bytes(size_t in_cap) { return (n_tiles_for(in_cap + 16) + 1 + 5 * rec_capacity(in_cap) + SCAN_BLOCKS) * 4; }

int sam_transcode(const uint8_t* in, size_t n, bool final, uint8_t* out, void* scratch, size_t in_cap, Result* res, cudaStream_t st) {
  const Scratch s = carve(scratch, in_cap);
  const uint8_t* A = (const uint8_t*)((uintptr_t)in & ~(uintptr_t)15);
  const uint32_t lo = (uint32_t)(in - A), hi = lo + (uint32_t)n;
  const uint32_t tiles = (uint32_t)n_tiles_for(hi);
  cudaMemsetAsync(res, 0, sizeof(Result), st);
  if(!tiles) return 0;
  sam_count_kernel<<<tiles, TILE_THREADS, 0, st>>>(A, lo, hi, s.tile_cnt, res);
  sam_tiles_kernel<<<1, 1024, 0, st>>>(s.tile_cnt, tiles, (uint32_t)s.rec_cap, lo, hi, final ? 1u : 0u, res);
  sam_index_kernel<<<tiles, TILE_THREADS, 0, st>>>(A, lo, hi, s.tile_cnt, s.starts, (uint32_t)s.rec_cap);
  sam_parse_kernel<<<record_grid(), 256, 0, st>>>(A, lo, hi, final ? 1u : 0u, s.starts, res, s.seq, s.qual, s.len);
  return 4 + scan_and_emit(A, false, s, out, res, st);
}

int bam_transcode(const uint8_t* in, size_t n, const uint32_t* offs, uint32_t n_recs, uint8_t* out, void* scratch, size_t in_cap,
                  Result* res, cudaStream_t st) {
  (void)n;
  const Scratch s = carve(scratch, in_cap);
  const uint8_t* A = (const uint8_t*)((uintptr_t)in & ~(uintptr_t)15);
  const uint32_t lo = (uint32_t)(in - A);
  cudaMemsetAsync(res, 0, sizeof(Result), st);
  if(!n_recs) return 0;
  bam_parse_kernel<<<(n_recs + 255) / 256, 256, 0, st>>>(A, lo, offs, n_recs, res, s.seq, s.qual, s.len);
  return 1 + scan_and_emit(A, true, s, out, res, st);
}

}  // namespace jfsam
