// jf_cli.cc -- `jellyfish-b200`: the host driver that keeps the reference's command line
// for the count path and calls the sm_90a engine through the C ABI (include/jfgpu.h).
//
//   jellyfish-b200 count  ...   switches of sub_commands/count_main_cmdline.yaggo:4-112
//   jellyfish-b200 dump   ...   sub_commands/dump_main_cmdline.yaggo  (CPU reader of the format)
//   jellyfish-b200 query  ...   sub_commands/query_main_cmdline.yaggo (-s on the GPU when there is one, else a CPU reader)
//   jellyfish-b200 info / histo / stats / merge      small CPU readers used by the tests
//
// The flow of `count` mirrors count_main (sub_commands/count_main.cc:218-385): header
// fill_standard + cmdline, build the table, stream the input files, dump, --timing.
#include <errno.h>
#include <fcntl.h>
#include <getopt.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <unistd.h>

#include <algorithm>
#include <chrono>
#include <condition_variable>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <functional>
#include <iostream>
#include <limits>
#include <map>
#include <mutex>
#include <queue>
#include <string>
#include <thread>
#include <vector>

#include "jfgpu.h"
#include "jf_file_header.hpp"
#include "jf_inputs.hpp"

namespace {

[[noreturn]] void die(const std::string& msg) {
  std::cerr << msg << std::endl;
  exit(EXIT_FAILURE);
}
[[noreturn]] void usage_error(const std::string& msg) {
  std::cerr << "Error: " << msg << std::endl;
  exit(EXIT_FAILURE);
}

// SI suffixes, powers of 1000 (doc/jellyfish.man:137-139)
uint64_t parse_u64(const char* s, bool suffix, const char* name) {
  errno = 0;
  char* end = nullptr;
  while(*s == ' ') ++s;
  if(*s == '-') usage_error(std::string("Invalid negative value for switch ") + name);
  unsigned long long v = strtoull(s, &end, 0);
  if(errno || end == s) usage_error(std::string("Invalid numeric value '") + s + "' for switch " + name);
  if(*end) {
    uint64_t mult = 0;
    if(suffix && end[1] == '\0') switch(*end) {
      case 'k': mult = 1000ULL; break;
      case 'M': mult = 1000000ULL; break;
      case 'G': mult = 1000000000ULL; break;
      case 'T': mult = 1000000000000ULL; break;
      case 'P': mult = 1000000000000000ULL; break;
      case 'E': mult = 1000000000000000000ULL; break;
    }
    if(!mult) usage_error(std::string("Invalid numeric value '") + s + "' for switch " + name);
    v *= mult;
  }
  return v;
}

// 2-bit packed k-mer <-> text: first base in the most significant pair (mer_dna.hpp:451-462,525-542).  A key is held in
// MER_WORDS 64-bit words, word 0 least significant, whatever k (up to 128)
constexpr unsigned MER_WORDS = 4;
std::string mer_to_string(const uint64_t* w, unsigned k) {
  std::string s(k, 'A');
  for(unsigned i = 0; i < k; ++i) {
    unsigned bit = 2 * (k - 1 - i);
    s[i] = "ACGT"[(w[bit >> 6] >> (bit & 63)) & 3];
  }
  return s;
}
bool string_to_mer(const char* s, unsigned k, uint64_t* w) {
  std::fill(w, w + MER_WORDS, 0);
  if(strlen(s) != k) return false;
  for(unsigned i = 0; i < k; ++i) {
    int c;
    switch(s[i]) { case 'A': case 'a': c = 0; break; case 'C': case 'c': c = 1; break;
                   case 'G': case 'g': c = 2; break; case 'T': case 't': c = 3; break; default: return false; }
    unsigned bit = 2 * (k - 1 - i);
    w[bit >> 6] |= (uint64_t)c << (bit & 63);
  }
  return true;
}
void reverse_complement(const uint64_t* in, unsigned k, uint64_t* out) {
  std::fill(out, out + MER_WORDS, 0);
  for(unsigned i = 0; i < k; ++i) {
    unsigned bit = 2 * i;
    uint64_t c = 3 - ((in[bit >> 6] >> (bit & 63)) & 3);
    unsigned ob = 2 * (k - 1 - i);
    out[ob >> 6] |= c << (ob & 63);
  }
}
bool mer_less(const uint64_t* a, const uint64_t* b) {
  for(int q = MER_WORDS - 1; q > 0; --q) if(a[q] != b[q]) return a[q] < b[q];
  return a[0] < b[0];
}
bool mer_equal(const uint64_t* a, const uint64_t* b) { return std::equal(a, a + MER_WORDS, b); }

// ------------------------------------------------------------------------------------------
// reader of the binary/sorted format (binary_dumper.hpp:83-109)
// ------------------------------------------------------------------------------------------
struct db_reader {
  jfb::file_header header;
  const unsigned char* base = nullptr;   // mmap
  size_t file_size = 0, body_off = 0, n_records = 0;
  unsigned k = 0, key_bytes = 0, counter_len = 0, rec = 0;
  jfb::gf2_matrix matrix;
  uint64_t size_mask = 0;
  int fd = -1;

  void open(const char* path) {
    fd = ::open(path, O_RDONLY);
    if(fd < 0) die(std::string("Failed to open input file '") + path + "'");
    struct stat st;
    if(fstat(fd, &st) != 0) die(std::string("Can't stat file '") + path + "'");
    file_size = st.st_size;
    base = file_size ? (const unsigned char*)mmap(nullptr, file_size, PROT_READ, MAP_PRIVATE, fd, 0) : nullptr;
    if(file_size && base == MAP_FAILED) die(std::string("Can't mmap file '") + path + "'");
    if(!header.read((const char*)base, file_size)) die(std::string("Failed to parse header of file '") + path + "'");
    body_off = header.offset();
    k = header.key_len() / 2;
    key_bytes = (header.key_len() + 7) / 8;
    counter_len = header.counter_len();
    rec = key_bytes + counter_len;
    if(header.format() == "binary/sorted" || header.format() == "text/sorted") {
      matrix = header.matrix(1);
      size_mask = header.size() - 1;
    }
    if(header.format() == "binary/sorted") n_records = rec ? (file_size - body_off) / rec : 0;
  }
  void key_at(size_t i, uint64_t* w) const {
    std::fill(w, w + MER_WORDS, 0);
    memcpy(w, base + body_off + i * rec, key_bytes);
  }
  uint64_t val_at(size_t i) const {
    uint64_t v = 0;
    memcpy(&v, base + body_off + i * rec + key_bytes, counter_len);
    return v;
  }
  uint64_t pos_of(const uint64_t* w) const { return matrix.times(w) & size_mask; }
  ~db_reader() { if(base && base != MAP_FAILED) munmap((void*)base, file_size); if(fd >= 0) close(fd); }
};

// ------------------------------------------------------------------------------------------
// count
// ------------------------------------------------------------------------------------------
struct count_args {
  uint32_t mer_len = 0; bool mer_len_given = false;
  uint64_t size = 0; bool size_given = false;
  uint32_t threads = 1, Files = 1, Generators = 1;
  const char* output = "mer_counts.jf";
  uint32_t counter_len = 7, out_counter_len = 4, reprobes = 126;
  bool canonical = false, text = false, disk = false, no_merge = false, no_unlink = false, no_write = false;
  bool bc_given = false, bf_size_given = false, if_given = false, generator_given = false, sam_given = false;
  bool qual_given = false, timing_given = false, lower_given = false, upper_given = false;
  bool min_qual_char_given = false, min_quality_given = false;
  std::string min_qual_char; int quality_start = 64, min_quality = 0; uint32_t min_qual = 0;
  uint64_t bf_size = 0, lower = 0, upper = 0;
  double bf_fp = 0.01;
  const char* timing = "";
  const char* bc_path = nullptr;
  int device = 0;
  std::vector<const char*> files;
  std::vector<const char*> if_files;
  std::vector<const char*> sam_files;  // --sam, counted after the other inputs (stream_manager.hpp:134-145)
  jfb::generator_spec gen;             // -g / -G / -S
};

struct sink_ctx { FILE* f; bool ok; bool text; unsigned k, key_bytes, rec; };
int file_sink(void* ctx, const void* recs, size_t n) {
  sink_ctx* c = (sink_ctx*)ctx;
  if(!c->text) {
    if(fwrite(recs, 1, n, c->f) != n) { c->ok = false; return 1; }
    return 0;
  }
  // --text (text_dumper.hpp: "MER count" lines, counts not clipped): records arrive with 8-byte counters
  const unsigned char* p = (const unsigned char*)recs;
  std::string line;
  for(size_t off = 0; off + c->rec <= n; off += c->rec) {
    uint64_t w[MER_WORDS] = {0, 0, 0, 0}, v = 0;
    memcpy(w, p + off, c->key_bytes);
    memcpy(&v, p + off + c->key_bytes, 8);
    line = mer_to_string(w, c->k);
    line += ' '; line += std::to_string((unsigned long long)v); line += '\n';
    if(fwrite(line.data(), 1, line.size(), c->f) != line.size()) { c->ok = false; return 1; }
  }
  return 0;
}

// ---- stream the inputs through an engine: a reader thread fills pinned buffers, the caller's thread feeds them (host/jf_inputs.hpp) ----
void stream_files(jfgpu_handle h, const std::vector<const char*>& file_list, const jfb::generator_spec& gen = jfb::generator_spec(),
                  const std::vector<const char*>& sam_files = {}) {
  static_assert((uint32_t)jfb::INPUT_FILE_BEGIN == (uint32_t)JFGPU_FILE_BEGIN && (uint32_t)jfb::INPUT_FILE_END == (uint32_t)JFGPU_FILE_END &&
                (uint32_t)jfb::INPUT_FORMAT_SAM == (uint32_t)JFGPU_FORMAT_SAM && (uint32_t)jfb::INPUT_FORMAT_BAM == (uint32_t)JFGPU_FORMAT_BAM,
                "chunk flags are the engine's");
  jfb::input_buffers mem = { [](size_t n) { return jfgpu_host_alloc(n); }, [](void* p) { jfgpu_host_free(p); } };
  const std::string err = jfb::stream_inputs(file_list, gen, mem,
    [&](const char* data, size_t n, uint32_t flags) { return jfgpu_feed(h, data, n, flags); },
    [&]() { return std::string(jfgpu_last_error(h)); }, (size_t)64 << 20, sam_files);
  if(!err.empty()) die(err);
}

// `inputs`: the byte stream `count` / `bc` would hand to the engine for these arguments (files, then the outputs of the -g
// commands, then the --sam files inflated), on standard output; --marks lists the chunks and their flags on standard error.
// Needs no device: a way to look at what a set of generator commands or a compressed --sam file really produces.
int inputs_main(int argc, char* argv[]) {
  jfb::generator_spec gen;
  std::vector<const char*> sam_files;
  bool marks = false; size_t chunk_bytes = (size_t)64 << 20;
  enum { O_MARKS = 1000, O_CHUNK, O_SAM };
  static struct option longs[] = {
    {"generator", required_argument, 0, 'g'}, {"Generators", required_argument, 0, 'G'}, {"shell", required_argument, 0, 'S'},
    {"marks", no_argument, 0, O_MARKS}, {"chunk", required_argument, 0, O_CHUNK}, {"sam", required_argument, 0, O_SAM}, {0, 0, 0, 0} };
  optind = 1; int c;
  while((c = getopt_long(argc, argv, "g:G:S:", longs, 0)) != -1) switch(c) {
    case 'g': gen.cmds_path = optarg; break;
    case 'G': gen.concurrent = (uint32_t)parse_u64(optarg, false, "-G"); break;
    case 'S': gen.shell = optarg; break;
    case O_MARKS: marks = true; break;
    case O_CHUNK: chunk_bytes = (size_t)parse_u64(optarg, true, "--chunk"); if(chunk_bytes == 0) usage_error("--chunk must be positive"); break;
    case O_SAM: sam_files.push_back(optarg); break;
    default: usage_error("Usage: jellyfish-b200 inputs [-g path] [-G n] [-S shell] [--sam path] [--marks] [--chunk bytes] file:path*");
  }
  std::vector<const char*> files;
  for(int i = optind; i < argc; ++i) files.push_back(argv[i]);
  jfb::input_buffers mem = { [](size_t n) { return malloc(n); }, [](void* p) { free(p); } };
  std::string werr;
  const std::string err = jfb::stream_inputs(files, gen, mem,
    [&](const char* data, size_t n, uint32_t flags) -> int {
      if(marks) std::cerr << "chunk " << n << (flags & JFGPU_FILE_BEGIN ? " begin" : "") << (flags & JFGPU_FILE_END ? " end" : "")
                          << (flags & JFGPU_FORMAT_SAM ? " sam" : "") << (flags & JFGPU_FORMAT_BAM ? " bam" : "") << "\n";
      if(n && fwrite(data, 1, n, stdout) != n) { werr = "Error writing the standard output"; return 1; }
      return 0;
    },
    [&]() { return werr; }, chunk_bytes, sam_files);
  fflush(stdout);
  if(!err.empty()) die(err);
  return 0;
}

// load_bloom_filter (sub_commands/count_main.cc:191-206): header checks, then the counter bytes go to the device
void load_bloom_counter(jfgpu_handle h, const char* path, unsigned mer_len) {
  int fd = ::open(path, O_RDONLY);
  if(fd < 0) die(std::string("Failed to open bloom filter file '") + path + "'");
  struct stat st;
  if(fstat(fd, &st) != 0) die(std::string("Can't stat file '") + path + "'");
  const size_t size = st.st_size;
  const char* base = size ? (const char*)mmap(nullptr, size, PROT_READ, MAP_PRIVATE, fd, 0) : nullptr;
  if(size && base == MAP_FAILED) die(std::string("Can't mmap file '") + path + "'");
  jfb::file_header hd;
  if(!hd.read(base, size)) die(std::string("Failed to parse bloom filter file '") + path + "'");
  if(hd.format() != "bloomcounter") die(std::string("Invalid format '") + hd.format() + "'. Expected 'bloomcounter'");
  if(hd.key_len() != mer_len * 2) die("Invalid mer length in bloom filter");
  const jfb::gf2_matrix m1 = hd.matrix(1), m2 = hd.matrix(2);
  std::vector<uint64_t> c1(2 * mer_len), c2(2 * mer_len);
  for(unsigned i = 0; i < 2 * mer_len; ++i) { c1[i] = m1[i]; c2[i] = m2[i]; }
  if(jfgpu_bloom_load(h, hd.size(), (uint32_t)hd.nb_hashes(), c1.data(), c2.data(), base + hd.offset(), size - hd.offset()) != JFGPU_OK)
    die(std::string("Bloom filter file is truncated or invalid: ") + jfgpu_last_error(h));
  if(base) munmap((void*)base, size);
  ::close(fd);
}

// ------------------------------------------------------------------------------------------
// bc (sub_commands/bc_main.cc:84-161): build a Bloom counter of the k-mers of the input
// ------------------------------------------------------------------------------------------
int bc_main(int argc, char* argv[]) {
  using clk = std::chrono::system_clock;
  auto start_time = clk::now();
  jfb::file_header header;
  header.fill_standard();
  header.set_cmdline(argc, argv);
  uint32_t mer_len = 0; uint64_t size = 0; double fpr = 0.001; bool canonical = false, mer_given = false, size_given = false, timing_given = false;
  const char* output = "mer_bloom_filter"; const char* timing = ""; int device = 0;
  jfb::generator_spec gen;
  enum { O_TIMING = 1000, O_DEVICE };
  static struct option longs[] = {
    {"mer-len", required_argument, 0, 'm'}, {"size", required_argument, 0, 's'}, {"fpr", required_argument, 0, 'f'},
    {"threads", required_argument, 0, 't'}, {"Files", required_argument, 0, 'F'}, {"output", required_argument, 0, 'o'},
    {"canonical", no_argument, 0, 'C'}, {"timing", required_argument, 0, O_TIMING}, {"device", required_argument, 0, O_DEVICE},
    {"generator", required_argument, 0, 'g'}, {"Generators", required_argument, 0, 'G'}, {"shell", required_argument, 0, 'S'}, {0, 0, 0, 0} };
  optind = 1; int c;
  while((c = getopt_long(argc, argv, "m:s:f:t:F:o:Cg:G:S:", longs, 0)) != -1) switch(c) {
    case 'g': gen.cmds_path = optarg; break;
    case 'G': gen.concurrent = (uint32_t)parse_u64(optarg, false, "-G"); break;
    case 'S': gen.shell = optarg; break;
    case 'm': mer_len = (uint32_t)parse_u64(optarg, false, "-m"); mer_given = true; break;
    case 's': size = parse_u64(optarg, true, "-s"); size_given = true; break;
    case 'f': fpr = atof(optarg); break;
    case 't': case 'F': break;
    case 'o': output = optarg; break;
    case 'C': canonical = true; break;
    case O_TIMING: timing = optarg; timing_given = true; break;
    case O_DEVICE: device = atoi(optarg); break;
    default: usage_error("Usage: jellyfish-b200 bc [options] file:path+");
  }
  std::vector<const char*> files;
  for(int i = optind; i < argc; ++i) files.push_back(argv[i]);
  if(!mer_given) usage_error("Missing required switch --mer-len");
  if(!size_given) usage_error("Missing required switch --size");
  if(mer_len < 1 || mer_len > 64) usage_error("jellyfish-b200 bc supports mer lengths 1..64 (no Bloom counter for longer k-mers)");
  jfgpu_params p;
  memset(&p, 0, sizeof(p));
  p.struct_size = sizeof(p);
  p.k = mer_len; p.size = 1; p.counter_len = 7; p.canonical = canonical; p.device = device; p.n_shards = 1;
  p.bloom_counter = 1; p.bf_size = size; p.bf_fp = fpr;
  jfgpu_handle h = nullptr;
  if(jfgpu_create(&p, &h) != JFGPU_OK) die(std::string("Failed to create the device Bloom counter: ") + jfgpu_last_error(nullptr));
  jfgpu_bloom_info bi;
  if(jfgpu_bloom_info_get(h, &bi) != JFGPU_OK) die(jfgpu_last_error(h));
  header.canonical(canonical);
  std::ofstream out(output, std::ios::binary);
  if(!out.good()) die(std::string("Can't open output file '") + output + "'");
  header.format("bloomcounter");
  header.key_len(mer_len * 2);
  header.matrix(jfb::gf2_matrix(bi.matrix_r, bi.matrix_c, bi.matrix1), 1);
  header.matrix(jfb::gf2_matrix(bi.matrix_r, bi.matrix_c, bi.matrix2), 2);
  header.size(bi.m);
  header.nb_hashes(bi.nb_hashes);
  header.write(out);
  out.close();
  auto after_init_time = clk::now();
  stream_files(h, files, gen);
  if(jfgpu_finish(h, nullptr) != JFGPU_OK) die(jfgpu_last_error(h));
  auto after_count_time = clk::now();
  FILE* f = fopen(output, "ab");
  if(!f) die(std::string("Can't open output file '") + output + "'");
  sink_ctx sc = { f, true, false, mer_len, 0, 0 };
  int rc = jfgpu_bloom_dump(h, file_sink, &sc);
  fclose(f);
  if(rc != JFGPU_OK || !sc.ok) die(std::string("Error while writing the Bloom counter: ") + jfgpu_last_error(h));
  auto after_dump_time = clk::now();
  if(timing_given) {
    auto secs = [](clk::duration d) { return std::chrono::duration_cast<std::chrono::duration<double>>(d).count(); };
    std::ofstream tf(timing);
    tf << "Init     " << secs(after_init_time - start_time) << "\n"
       << "Counting " << secs(after_count_time - after_init_time) << "\n"
       << "Writing  " << secs(after_dump_time - after_count_time) << "\n";
  }
  jfgpu_destroy(h);
  return 0;
}

// k-way SUM merge of binary/sorted files into `output` under header `oh` (defined with merge_main below)
enum merge_op { MERGE_SUM, MERGE_MIN, MERGE_MAX, MERGE_JACCARD };      // merge_files.hpp: SUM, MIN, MAX, JACCARD
void merge_dbs(const std::vector<std::string>& inputs, const char* output, jfb::file_header& oh, uint64_t lower, uint64_t upper, merge_op op = MERGE_SUM);

int count_main(int argc, char* argv[]) {
  using clk = std::chrono::system_clock;
  auto start_time = clk::now();
  jfb::file_header header;
  header.fill_standard();
  header.set_cmdline(argc, argv);

  count_args a;
  enum { O_SAM = 1000, O_OCL, O_BC, O_BFSIZE, O_BFFP, O_IF, O_QSTART, O_MINQ, O_TEXT, O_DISK, O_NOMERGE, O_NOUNLINK,
         O_TIMING, O_NOWRITE, O_DEVICE };
  static struct option longs[] = {
    {"mer-len", required_argument, 0, 'm'}, {"size", required_argument, 0, 's'}, {"threads", required_argument, 0, 't'},
    {"sam", required_argument, 0, O_SAM}, {"Files", required_argument, 0, 'F'}, {"generator", required_argument, 0, 'g'},
    {"Generators", required_argument, 0, 'G'}, {"shell", required_argument, 0, 'S'}, {"output", required_argument, 0, 'o'},
    {"counter-len", required_argument, 0, 'c'}, {"out-counter-len", required_argument, 0, O_OCL},
    {"canonical", no_argument, 0, 'C'}, {"bc", required_argument, 0, O_BC}, {"bf-size", required_argument, 0, O_BFSIZE},
    {"bf-fp", required_argument, 0, O_BFFP}, {"if", required_argument, 0, O_IF}, {"min-qual-char", required_argument, 0, 'Q'},
    {"quality-start", required_argument, 0, O_QSTART}, {"min-quality", required_argument, 0, O_MINQ},
    {"reprobes", required_argument, 0, 'p'}, {"text", no_argument, 0, O_TEXT}, {"disk", no_argument, 0, O_DISK},
    {"no-merge", no_argument, 0, O_NOMERGE}, {"no-unlink", no_argument, 0, O_NOUNLINK},
    {"lower-count", required_argument, 0, 'L'}, {"upper-count", required_argument, 0, 'U'},
    {"timing", required_argument, 0, O_TIMING}, {"no-write", no_argument, 0, O_NOWRITE},
    {"device", required_argument, 0, O_DEVICE}, {"help", no_argument, 0, 'h'}, {0, 0, 0, 0} };
  optind = 1;
  int c;
  while((c = getopt_long(argc, argv, "m:s:t:F:g:G:S:o:c:CQ:p:L:U:h", longs, 0)) != -1) {
    switch(c) {
    case 'm': a.mer_len = (uint32_t)parse_u64(optarg, false, "-m"); a.mer_len_given = true; break;
    case 's': a.size = parse_u64(optarg, true, "-s"); a.size_given = true; break;
    case 't': a.threads = (uint32_t)parse_u64(optarg, false, "-t"); break;
    case 'F': a.Files = (uint32_t)parse_u64(optarg, false, "-F"); break;
    case 'g': a.generator_given = true; a.gen.cmds_path = optarg; break;
    case 'G': a.Generators = (uint32_t)parse_u64(optarg, false, "-G"); a.gen.concurrent = a.Generators; break;
    case 'S': a.gen.shell = optarg; break;
    case 'o': a.output = optarg; break;
    case 'c': a.counter_len = (uint32_t)parse_u64(optarg, false, "-c"); break;
    case O_OCL: a.out_counter_len = (uint32_t)parse_u64(optarg, false, "--out-counter-len"); break;
    case 'C': a.canonical = true; break;
    case O_BC: a.bc_given = true; a.bc_path = optarg; break;
    case O_SAM: a.sam_given = true; a.sam_files.push_back(optarg); break;
    case O_BFSIZE: a.bf_size = parse_u64(optarg, true, "--bf-size"); a.bf_size_given = true; break;
    case O_BFFP: a.bf_fp = atof(optarg); break;
    case O_IF: a.if_given = true; a.if_files.push_back(optarg); break;
    case 'Q': a.min_qual_char = optarg; a.min_qual_char_given = true; break;
    case O_QSTART: a.quality_start = atoi(optarg); break;
    case O_MINQ: a.min_quality = atoi(optarg); a.min_quality_given = true; break;
    case 'p': a.reprobes = (uint32_t)parse_u64(optarg, false, "-p"); break;
    case O_TEXT: a.text = true; break;
    case O_DISK: a.disk = true; break;
    case O_NOMERGE: a.no_merge = true; break;
    case O_NOUNLINK: a.no_unlink = true; break;
    case 'L': a.lower = parse_u64(optarg, false, "-L"); a.lower_given = true; break;
    case 'U': a.upper = parse_u64(optarg, false, "-U"); a.upper_given = true; break;
    case O_TIMING: a.timing = optarg; a.timing_given = true; break;
    case O_NOWRITE: a.no_write = true; break;
    case O_DEVICE: a.device = atoi(optarg); break;
    case 'h': std::cout << "Usage: jellyfish-b200 count [options] file:path+\n"; return 0;
    default: usage_error("Invalid command line. Usage: jellyfish-b200 count [options] file:path+");
    }
  }
  for(int i = optind; i < argc; ++i) a.files.push_back(argv[i]);
  if(!a.mer_len_given) usage_error("Missing required switch --mer-len");
  if(!a.size_given) usage_error("Missing required switch --size");
  if(a.bc_given && a.bf_size_given) usage_error("Switches [--bf-size] and [--bc] conflict");
  // count_main.cc:234-256
  if(a.min_qual_char_given) {
    if(a.min_qual_char.size() != 1) usage_error("[-Q, --min-qual-char] must be one character.");
    const char c = a.min_qual_char[0];
    if(c < '!' || c > '~') usage_error(std::string("Quality character '") + c + "' is outside of the range [!, ~]");
    a.min_qual = (uint32_t)(unsigned char)c;
  }
  if(a.min_quality_given) {
    if(a.quality_start < '!' || a.quality_start > '~') usage_error("Quality start " + std::to_string(a.quality_start) + " is outside the range [33, 126]");
    const int mq = a.quality_start + a.min_quality;
    if(mq < '!' || mq > '~') usage_error("Min quality " + std::to_string(a.min_quality) + " is outside the range [0, " + std::to_string((int)'~' - a.quality_start) + "]");
    a.min_qual = (uint32_t)mq;
  }
  a.qual_given = a.min_qual != 0;
  if(a.disk && a.text) usage_error("--disk with --text is not supported by jellyfish-b200 (intermediate files are binary)");
  if(a.mer_len < 1 || a.mer_len > 128) usage_error("jellyfish-b200 supports mer lengths 1..128");
  if(a.mer_len > 64 && (a.bf_size_given || a.bc_given)) usage_error("--bf-size and --bc take mer lengths up to 64");

  header.canonical(a.canonical);
  jfgpu_params p;
  memset(&p, 0, sizeof(p));
  p.struct_size = sizeof(p);
  p.k = a.mer_len; p.size = a.size; p.counter_len = a.counter_len; p.max_reprobe = a.reprobes;
  p.canonical = a.canonical; p.allow_regrow = a.disk ? 0 : 1; p.device = a.device;      // --disk: no size doubling (count_main.cc:277) p.shard_index = 0; p.n_shards = 1;
  if(a.bf_size_given) { p.bf_size = a.bf_size; p.bf_fp = a.bf_fp; }       // count_main.cc:317-321
  p.min_qual = a.min_qual;                                                 // count_main.cc:326-329
  jfgpu_handle h = nullptr;
  if(jfgpu_create(&p, &h) != JFGPU_OK) die(std::string("Failed to create the device hash: ") + jfgpu_last_error(nullptr));
  // header + sorted records of the resident table into `path`; `final`: the one output file (-L/-U apply), else an
  // intermediate file of --disk (everything, merged later)
  auto write_table = [&](const char* path, bool final) {
    jfgpu_table_info ti;
    jfgpu_table_info_get(h, &ti);
    header.size(ti.size);
    header.key_len(ti.key_len);
    header.val_len(ti.val_len);
    if(ti.matrix_identity) header.matrix(ti.matrix_r == ti.matrix_c ? jfb::gf2_matrix::identity(ti.matrix_c)
                                                                      : jfb::gf2_matrix::low_identity(ti.matrix_r, ti.matrix_c));
    else header.matrix(jfb::gf2_matrix(ti.matrix_r, ti.matrix_c, ti.matrix_columns));
    header.max_reprobe(ti.max_reprobe);
    header.set_reprobes(ti.reprobes);
    if(a.text) header.format("text/sorted");
    else { header.format("binary/sorted"); header.counter_len(a.out_counter_len); }
    std::ofstream out(path, std::ios::binary);
    if(!out.good()) die(std::string("Can't open output file '") + path + "'");
    header.write(out);
    out.close();
    FILE* f = fopen(path, "ab");
    if(!f) die(std::string("Can't open output file '") + path + "'");
    std::vector<char> iobuf((size_t)8 << 20);
    setvbuf(f, iobuf.data(), _IOFBF, iobuf.size());
    const unsigned key_bytes = (2 * a.mer_len + 7) / 8;
    sink_ctx sc = { f, true, a.text, a.mer_len, key_bytes, key_bytes + 8 };
    const uint64_t lo = final && a.lower_given ? a.lower : 0, hi = final && a.upper_given ? a.upper : std::numeric_limits<uint64_t>::max();
    int rc = jfgpu_dump(h, lo, hi, a.text ? 8 : a.out_counter_len, file_sink, &sc, nullptr);
    fclose(f);
    if(rc != JFGPU_OK) die(std::string("Error while dumping: ") + jfgpu_last_error(h));
  };
  // --disk (hash_counter.hpp:187-192, dumper.hpp:45-60): a full table is written to <output>0, <output>1, ... and zeroed
  struct spill_state { std::vector<std::string> files; std::function<void(const char*)> write; const char* prefix; } spill;
  spill.prefix = a.output;
  spill.write = [&](const char* path) { write_table(path, false); };
  if(a.disk) {
    auto hook = [](void* ctx, jfgpu_handle) -> int {
      spill_state* sp = (spill_state*)ctx;
      const std::string name = std::string(sp->prefix) + std::to_string(sp->files.size());
      sp->files.push_back(name);
      sp->write(name.c_str());
      return 0;
    };
    if(jfgpu_set_spill(h, hook, &spill) != JFGPU_OK) die(jfgpu_last_error(h));
  }
  auto after_init_time = clk::now();

  // count_main.cc:288-295: with --if the keys of those files are primed first, then only they are counted
  if(a.if_given) {
    if(jfgpu_set_op(h, JFGPU_OP_PRIME) != JFGPU_OK) die(jfgpu_last_error(h));
    stream_files(h, a.if_files);
    if(jfgpu_set_op(h, JFGPU_OP_UPDATE) != JFGPU_OK) die(jfgpu_last_error(h));
  }
  if(a.bc_given) load_bloom_counter(h, a.bc_path, a.mer_len);                 // count_main.cc:311-315
  stream_files(h, a.files, a.gen, a.sam_files);   // files, the outputs of the -g commands, the --sam files (count_main.cc:297-303)
  jfgpu_stats st;
  if(jfgpu_finish(h, &st) != JFGPU_OK) die(jfgpu_last_error(h));
  auto after_count_time = clk::now();

  // ---- dump (binary_dumper::_dump -> sorted_dumper::_dump, binary_dumper.hpp:62-69) ------------
  if(!a.no_write) {
    if(spill.files.empty()) write_table(a.output, true);
    else {
      // intermediate files exist (--disk): the rest of the table becomes one more, then a round of merging (count_main.cc:356-371)
      const std::string last = std::string(a.output) + std::to_string(spill.files.size());
      spill.files.push_back(last);
      write_table(last.c_str(), false);
      if(!a.no_merge) {
        const uint64_t lo = a.lower_given ? a.lower : 0, hi = a.upper_given ? a.upper : std::numeric_limits<uint64_t>::max();
        merge_dbs(spill.files, a.output, header, lo, hi);
        if(!a.no_unlink) for(const std::string& f : spill.files) unlink(f.c_str());
      }
    }
  }
  auto after_dump_time = clk::now();
  if(a.timing_given) {
    auto secs = [](clk::duration d) { return std::chrono::duration_cast<std::chrono::duration<double>>(d).count(); };
    std::ofstream tf(a.timing);
    tf << "Init     " << secs(after_init_time - start_time) << "\n"
       << "Counting " << secs(after_count_time - after_init_time) << "\n"
       << "Writing  " << secs(after_dump_time - after_count_time) << "\n";
  }
  jfgpu_destroy(h);
  return 0;
}

// ------------------------------------------------------------------------------------------
// dump (sub_commands/dump_main.cc:35-88)
// ------------------------------------------------------------------------------------------
int dump_main(int argc, char* argv[]) {
  bool column = false, tab = false, lower_given = false, upper_given = false;
  uint64_t lower = 0, upper = std::numeric_limits<uint64_t>::max();
  const char* output = nullptr;
  static struct option longs[] = { {"column", no_argument, 0, 'c'}, {"tab", no_argument, 0, 't'},
    {"lower-count", required_argument, 0, 'L'}, {"upper-count", required_argument, 0, 'U'},
    {"output", required_argument, 0, 'o'}, {0, 0, 0, 0} };
  optind = 1; int c;
  while((c = getopt_long(argc, argv, "ctL:U:o:", longs, 0)) != -1) switch(c) {
    case 'c': column = true; break; case 't': tab = true; break;
    case 'L': lower = parse_u64(optarg, false, "-L"); lower_given = true; break;
    case 'U': upper = parse_u64(optarg, false, "-U"); upper_given = true; break;
    case 'o': output = optarg; break;
    default: usage_error("Usage: jellyfish-b200 dump [options] db:path");
  }
  (void)lower_given; (void)upper_given;
  if(argc - optind != 1) usage_error("Requires exactly 1 argument.");
  db_reader db; db.open(argv[optind]);
  if(db.header.format() != "binary/sorted") die("Unknown format '" + db.header.format() + "'");
  FILE* out = output ? fopen(output, "w") : stdout;
  if(!out) die(std::string("Error opening output file '") + output + "'");
  uint64_t w[MER_WORDS];
  for(size_t i = 0; i < db.n_records; ++i) {
    uint64_t v = db.val_at(i);
    if(v < lower || v > upper) continue;
    db.key_at(i, w);
    std::string s = mer_to_string(w, db.k);
    if(column) fprintf(out, "%s%c%llu\n", s.c_str(), tab ? '\t' : ' ', (unsigned long long)v);
    else fprintf(out, ">%llu\n%s\n", (unsigned long long)v, s.c_str());
  }
  if(output) fclose(out);
  return 0;
}

// ------------------------------------------------------------------------------------------
// query (sub_commands/query_main.cc:86-123; binary_dumper.hpp:148-189): the file is sorted by
// (position, key), so a plain binary search on that pair finds a k-mer.
// ------------------------------------------------------------------------------------------
uint64_t db_lookup(const db_reader& db, const uint64_t* key) {
  const uint64_t pos = db.pos_of(key);
  size_t lo = 0, hi = db.n_records;
  uint64_t w[MER_WORDS];
  while(lo < hi) {
    size_t mid = lo + (hi - lo) / 2;
    db.key_at(mid, w);
    uint64_t mp = db.pos_of(w);
    bool less = mp != pos ? mp < pos : mer_less(w, key);
    if(less) lo = mid + 1; else hi = mid;
  }
  if(lo < db.n_records) { db.key_at(lo, w); if(mer_equal(w, key)) return db.val_at(lo); }
  return 0;
}

// query -s on the device (query_from_sequence, query_main.cc:45-51): the database's records go into a table of this GPU (its own
// hash matrix, twice as many slots as records), then every -s file streams through jfgpu_query into `out`
void query_sequences_device(const db_reader& db, const std::vector<const char*>& sequences, FILE* out) {
  jfgpu_params p;
  memset(&p, 0, sizeof(p));
  p.struct_size = sizeof(p);
  p.k = db.k; p.size = std::max<uint64_t>(2 * (uint64_t)db.n_records, 2); p.counter_len = 7; p.max_reprobe = 126;
  p.canonical = db.header.canonical(); p.allow_regrow = 1; p.n_shards = 1;
  jfgpu_handle h = nullptr;
  if(jfgpu_create(&p, &h) != JFGPU_OK) die(std::string("Failed to create the device hash: ") + jfgpu_last_error(nullptr));
  const size_t slice = std::max<size_t>(((size_t)1 << 30) / db.rec, 1) * db.rec;      // whole records of the mapped body
  const size_t body = db.n_records * db.rec;
  for(size_t off = 0; off < body; off += slice)
    if(jfgpu_load_records(h, db.base + db.body_off + off, std::min(slice, body - off), db.counter_len) != JFGPU_OK)
      die(std::string("Failed to load the database into the device hash: ") + jfgpu_last_error(h));
  bool write_ok = true;                         // (the engine hands over up to 64 MB of lines at a time: large fwrites)
  auto sink = [](void* ctx, const void* lines, size_t n) -> int {
    std::pair<FILE*, bool*>* c = (std::pair<FILE*, bool*>*)ctx;
    if(fwrite(lines, 1, n, c->first) != n) { *c->second = false; return 1; }
    return 0;
  };
  std::pair<FILE*, bool*> sc(out, &write_ok);
  jfb::input_buffers mem = { [](size_t n) { return jfgpu_host_alloc(n); }, [](void* q) { jfgpu_host_free(q); } };
  const std::string err = jfb::stream_inputs(sequences, jfb::generator_spec(), mem,
    [&](const char* data, size_t n, uint32_t flags) { return jfgpu_query(h, data, n, flags, sink, &sc, nullptr); },
    [&]() { return std::string(write_ok ? jfgpu_last_error(h) : "Error writing the query output"); });
  if(!err.empty()) die(err);
  if(fflush(out) != 0) die("Error writing the query output");
  jfgpu_destroy(h);
}

int query_main(int argc, char* argv[]) {
  std::vector<const char*> sequences; const char* output = nullptr; bool interactive = false;
  static struct option longs[] = { {"sequence", required_argument, 0, 's'}, {"output", required_argument, 0, 'o'},
    {"interactive", no_argument, 0, 'i'}, {"load", no_argument, 0, 'l'}, {"no-load", no_argument, 0, 'L'}, {0, 0, 0, 0} };
  optind = 1; int c;
  while((c = getopt_long(argc, argv, "s:o:ilL", longs, 0)) != -1) switch(c) {
    case 's': sequences.push_back(optarg); break; case 'o': output = optarg; break; case 'i': interactive = true; break;
    case 'l': case 'L': break;
    default: usage_error("Usage: jellyfish-b200 query [options] file:path mers:string*");
  }
  if(argc - optind < 1) usage_error("Requires at least 1 argument.");
  db_reader db; db.open(argv[optind]);
  if(db.header.format() != "binary/sorted") die("Unsupported format '" + db.header.format() + "'. Must be a bloom counter or binary list.");
  FILE* out = output ? fopen(output, "w") : stdout;
  if(!out) die(std::string("Error opening output file '") + output + "'");
  const bool canonical = db.header.canonical();
  auto query_one = [&](const char* s) {
    uint64_t m[MER_WORDS], r[MER_WORDS];
    if(!string_to_mer(s, db.k, m)) { fprintf(stderr, "Invalid mer '%s'\n", s); return; }
    const uint64_t* q = m;
    if(canonical) { reverse_complement(m, db.k, r); if(mer_less(r, m)) q = r; }
    fprintf(out, "%s %llu\n", mer_to_string(q, db.k).c_str(), (unsigned long long)db_lookup(db, q));
  };
  // every k-mer of the sequence files, in order: on the GPU when there is one, else with the binary search below
  const bool on_device = !sequences.empty() && jfgpu_device_count() > 0;
  if(on_device) query_sequences_device(db, sequences, out);
  if(!on_device) for(const char* path : sequences) {
    std::ifstream is(path);
    if(!is.good()) die(std::string("Can't open file '") + path + "'");
    std::string line, seq;
    auto flush = [&]() {
      uint64_t m[MER_WORDS] = {0, 0, 0, 0}, r[MER_WORDS] = {0, 0, 0, 0}; unsigned filled = 0;
      const unsigned k = db.k;
      for(char ch : seq) {
        int code;
        switch(ch) { case 'A': case 'a': code = 0; break; case 'C': case 'c': code = 1; break;
                     case 'G': case 'g': code = 2; break; case 'T': case 't': code = 3; break; default: code = -1; }
        if(code < 0) { filled = 0; continue; }
        // shift left m, shift right r
        for(int q = MER_WORDS - 1; q > 0; --q) m[q] = (m[q] << 2) | (m[q - 1] >> 62);
        m[0] = (m[0] << 2) | (uint64_t)code;
        const unsigned top = 2 * k;
        for(unsigned q = 0; q < MER_WORDS; ++q)
          if(top <= 64 * q) m[q] = 0; else if(top < 64 * (q + 1)) m[q] &= ((uint64_t)1 << (top - 64 * q)) - 1;
        for(unsigned q = 0; q + 1 < MER_WORDS; ++q) r[q] = (r[q] >> 2) | (r[q + 1] << 62);
        r[MER_WORDS - 1] >>= 2;
        unsigned ob = 2 * (k - 1); r[ob >> 6] |= (uint64_t)(3 - code) << (ob & 63);
        if(++filled >= k) {
          const uint64_t* q = (canonical && mer_less(r, m)) ? r : m;
          fprintf(out, "%s %llu\n", mer_to_string(q, k).c_str(), (unsigned long long)db_lookup(db, q));
        }
      }
      seq.clear();
    };
    while(std::getline(is, line)) {
      if(!line.empty() && line[0] == '>') { flush(); continue; }
      while(!line.empty() && (line.back() == '\r' || line.back() == '\n')) line.pop_back();
      seq += line;
    }
    flush();
  }
  for(int i = optind + 1; i < argc; ++i) query_one(argv[i]);
  if(interactive) { std::string s; while(std::cin >> s) query_one(s.c_str()); }
  if(output) fclose(out);
  return 0;
}

// ------------------------------------------------------------------------------------------
// info / histo / stats : sub_commands/{info,histo,stats}_main.cc
// ------------------------------------------------------------------------------------------
int info_main(int argc, char* argv[]) {
  bool skip = false, js = false, cmd = false;
  static struct option longs[] = { {"skip", no_argument, 0, 's'}, {"json", no_argument, 0, 'j'}, {"cmd", no_argument, 0, 'c'}, {0, 0, 0, 0} };
  optind = 1; int c;
  while((c = getopt_long(argc, argv, "sjc", longs, 0)) != -1) switch(c) {
    case 's': skip = true; break; case 'j': js = true; break; case 'c': cmd = true; break;
    default: usage_error("Usage: jellyfish-b200 info [options] file:path");
  }
  if(argc - optind != 1) usage_error("Requires exactly 1 argument.");
  db_reader db; db.open(argv[optind]);
  if(skip) { fwrite(db.base + db.body_off, 1, db.file_size - db.body_off, stdout); return 0; }
  if(js) { std::cout << db.header.root().dump() << "\n"; return 0; }
  std::vector<std::string> cl = db.header.cmdline();
  std::string line;
  for(size_t i = 0; i < cl.size(); ++i) { if(i) line += ' '; line += cl[i]; }
  if(cmd) { std::cout << line << "\n"; return 0; }
  const jfb::json& r = db.header.root();
  std::cout << "command: " << line << "\n"
            << "where: " << r.at("hostname").as_string() << ":" << r.at("pwd").as_string() << "\n"
            << "when: " << r.at("time").as_string() << "\n"
            << "canonical: " << (db.header.canonical() ? "yes" : "no") << "\n";
  return 0;
}

int histo_main(int argc, char* argv[]) {
  uint64_t low = 1, high = 10000, inc = 1; bool full = false; const char* output = nullptr;
  static struct option longs[] = { {"low", required_argument, 0, 'l'}, {"high", required_argument, 0, 'h'},
    {"increment", required_argument, 0, 'i'}, {"threads", required_argument, 0, 't'}, {"full", no_argument, 0, 'f'},
    {"output", required_argument, 0, 'o'}, {"buffer-size", required_argument, 0, 's'}, {"verbose", no_argument, 0, 'v'}, {0, 0, 0, 0} };
  optind = 1; int c;
  while((c = getopt_long(argc, argv, "l:h:i:t:fo:s:v", longs, 0)) != -1) switch(c) {
    case 'l': low = parse_u64(optarg, false, "-l"); break; case 'h': high = parse_u64(optarg, false, "-h"); break;
    case 'i': inc = parse_u64(optarg, false, "-i"); break; case 'f': full = true; break; case 'o': output = optarg; break;
    case 't': case 's': case 'v': break;
    default: usage_error("Usage: jellyfish-b200 histo [options] db:path");
  }
  if(argc - optind != 1) usage_error("Requires exactly 1 argument.");
  if(high < low) usage_error("High count value must be >= to low count value");
  db_reader db; db.open(argv[optind]);
  if(db.header.format() != "binary/sorted") die("Unknown format '" + db.header.format() + "'");
  // histo_main.cc:33-45,64-86
  const uint64_t base = inc >= low ? 0 : low - inc;
  const uint64_t ceil = high + inc;
  const uint64_t nb_buckets = (ceil + inc - base) / inc;
  std::vector<uint64_t> histo(nb_buckets, 0);
  for(size_t i = 0; i < db.n_records; ++i) {
    uint64_t v = db.val_at(i);
    if(v < base) ++histo[0];
    else if(v > ceil) ++histo[nb_buckets - 1];
    else ++histo[(v - base) / inc];
  }
  FILE* out = output ? fopen(output, "w") : stdout;
  if(!out) die(std::string("Error opening output file '") + output + "'");
  for(uint64_t i = 0, col = base; i < nb_buckets; ++i, col += inc)
    if(histo[i] > 0 || full) fprintf(out, "%llu %llu\n", (unsigned long long)col, (unsigned long long)histo[i]);
  if(output) fclose(out);
  return 0;
}

int stats_main(int argc, char* argv[]) {
  uint64_t lower = 0, upper = std::numeric_limits<uint64_t>::max(); const char* output = nullptr;
  static struct option longs[] = { {"recompute", no_argument, 0, 'r'}, {"lower-count", required_argument, 0, 'L'},
    {"upper-count", required_argument, 0, 'U'}, {"verbose", no_argument, 0, 'v'}, {"output", required_argument, 0, 'o'}, {0, 0, 0, 0} };
  optind = 1; int c;
  while((c = getopt_long(argc, argv, "rL:U:vo:", longs, 0)) != -1) switch(c) {
    case 'L': lower = parse_u64(optarg, false, "-L"); break; case 'U': upper = parse_u64(optarg, false, "-U"); break;
    case 'o': output = optarg; break; case 'r': case 'v': break;
    default: usage_error("Usage: jellyfish-b200 stats [options] db:path");
  }
  if(argc - optind != 1) usage_error("Requires exactly 1 argument.");
  db_reader db; db.open(argv[optind]);
  if(db.header.format() != "binary/sorted") die("Unknown format '" + db.header.format() + "'");
  uint64_t uniq = 0, distinct = 0, total = 0, maxc = 0;
  for(size_t i = 0; i < db.n_records; ++i) {
    uint64_t v = db.val_at(i);
    if(v < lower || v > upper) continue;
    if(v == 1) ++uniq;
    total += v; ++distinct; maxc = std::max(maxc, v);
  }
  FILE* out = output ? fopen(output, "w") : stdout;
  if(!out) die(std::string("Error opening output file '") + output + "'");
  fprintf(out, "Unique:    %llu\nDistinct:  %llu\nTotal:     %llu\nMax_count: %llu\n", (unsigned long long)uniq,
          (unsigned long long)distinct, (unsigned long long)total, (unsigned long long)maxc);
  if(output) fclose(out);
  return 0;
}

// ------------------------------------------------------------------------------------------
// merge (SUM only): k-way merge of files sharing size/matrix/key_len (jellyfish/merge_files.cc:45-176).
// This is how per-GPU shard dumps become one database.
// ------------------------------------------------------------------------------------------
int merge_main(int argc, char* argv[]) {
  const char* output = "mer_counts_merged.jf";
  uint64_t lower = 0, upper = std::numeric_limits<uint64_t>::max();
  bool lower_given = false, min_flag = false, max_flag = false, jaccard_flag = false;
  static struct option longs[] = { {"output", required_argument, 0, 'o'}, {"lower-count", required_argument, 0, 'L'},
    {"upper-count", required_argument, 0, 'U'}, {"min", no_argument, 0, 'm'}, {"max", no_argument, 0, 'M'}, {"jaccard", no_argument, 0, 'j'},
    {0, 0, 0, 0} };
  optind = 1; int c;
  while((c = getopt_long(argc, argv, "o:L:U:mMj", longs, 0)) != -1) switch(c) {
    case 'o': output = optarg; break;
    case 'L': lower = parse_u64(optarg, false, "-L"); lower_given = true; break; case 'U': upper = parse_u64(optarg, false, "-U"); break;
    case 'm': min_flag = true; break; case 'M': max_flag = true; break; case 'j': jaccard_flag = true; break;
    default: usage_error("Usage: jellyfish-b200 merge [options] input:string+");
  }
  if(min_flag && max_flag) usage_error("Switches [-M, --max] and [-m, --min] conflict");
  // merge_main.cc:31-37: with --min a k-mer absent from one input has count 0 and is left out unless -L says otherwise
  if(!lower_given && min_flag) lower = 1;
  merge_op op = MERGE_SUM;
  if(min_flag) op = MERGE_MIN;
  if(max_flag) op = MERGE_MAX;
  if(jaccard_flag) op = MERGE_JACCARD;
  const int n = argc - optind;
  if(n < 2) usage_error("Requires at least 2 arguments.");
  jfb::file_header oh;
  oh.fill_standard();
  oh.set_cmdline(argc, argv);
  std::vector<std::string> inputs;
  for(int i = 0; i < n; ++i) inputs.push_back(argv[optind + i]);
  merge_dbs(inputs, output, oh, lower, upper, op);          // (checks that the inputs go together)
  return 0;
}

// k-way merge in (position, key) order (merge_files.cc:44-104): per key the sum, the minimum (0 when an input lacks the key) or the
// maximum of the counts; JACCARD writes the two similarities instead of a database
void merge_dbs(const std::vector<std::string>& inputs, const char* output, jfb::file_header& oh, uint64_t lower, uint64_t upper, merge_op op) {
  const int n = (int)inputs.size();
  std::vector<db_reader> dbs(n);
  for(int i = 0; i < n; ++i) {
    dbs[i].open(inputs[i].c_str());
    const std::string& fmt = dbs[i].header.format();
    if(fmt != "binary/sorted" && fmt != "text/sorted") die(std::string("Unknown format '") + fmt + "'");
    if(i) {
      const jfb::file_header &a = dbs[0].header, &b = dbs[i].header;
      if(a.format() != b.format()) die(std::string("Can't merge files with different formats (") + a.format() + ", " + b.format() + ")");
      if(a.key_len() != b.key_len()) die("Can't merge hashes of different key lengths");
      if(a.size() != b.size()) die("Can't merge hash with different size");
      if(a.matrix(1) != b.matrix(1)) die("Can't merge hash with different hash function");
      if(a.max_reprobe_offset() != b.max_reprobe_offset()) die("Can't merge hashes with different reprobing strategies");
    }
  }
  const jfb::file_header& h0 = dbs[0].header;
  const bool text = h0.format() == "text/sorted";
  // exactly the keys merge_files() sets (merge_files.cc:125-138,160-165) on top of what the caller's header holds
  oh.size(h0.size()); oh.key_len(h0.key_len()); oh.matrix(h0.matrix(1));
  oh.max_reprobe(h0.max_reprobe()); { std::vector<uint64_t> r = h0.reprobes(); oh.set_reprobes(r.data()); }
  unsigned ocl_min = h0.counter_len();
  for(int i = 1; i < n; ++i) ocl_min = std::min<unsigned>(ocl_min, dbs[i].header.counter_len());
  oh.format(h0.format());
  if(!text) oh.counter_len(ocl_min);
  std::ofstream out(output, std::ios::binary);
  if(!out.good()) die(std::string("Can't open out file '") + output + "'");
  if(op != MERGE_JACCARD) oh.write(out);
  struct item { uint64_t pos; uint64_t key[MER_WORDS]; uint64_t val; int src; };
  auto greater = [](const item& a, const item& b) {
    if(a.pos != b.pos) return a.pos > b.pos;
    return mer_less(b.key, a.key);
  };
  std::priority_queue<item, std::vector<item>, decltype(greater)> heap(greater);
  // cursors: record index in a binary body; byte offset of the next "MER count" line in a text body (text_dumper.hpp:50-80)
  std::vector<size_t> cur(n, 0);
  const unsigned k = dbs[0].k;
  auto push = [&](int i) {
    item it; it.src = i;
    if(!text) {
      if(cur[i] >= dbs[i].n_records) return;
      dbs[i].key_at(cur[i], it.key); it.val = dbs[i].val_at(cur[i]); ++cur[i];
    } else {
      const char* p = (const char*)dbs[i].base + dbs[i].body_off + cur[i];
      const char* end = (const char*)dbs[i].base + dbs[i].file_size;
      while(p < end && (*p == '\n' || *p == ' ' || *p == '\t' || *p == '\r')) ++p;
      if(p >= end) return;
      const char* nl = (const char*)memchr(p, '\n', (size_t)(end - p));
      const char* stop = nl ? nl : end;
      std::string mer(p, std::min<size_t>(k, (size_t)(stop - p)));
      char* num_end = nullptr;
      const std::string num(p + mer.size(), (size_t)(stop - p) - mer.size());        // (a copy: the mapping may end right behind the line)
      it.val = strtoull(num.c_str(), &num_end, 10);
      if(!string_to_mer(mer.c_str(), k, it.key) || num_end == num.c_str())
        die(std::string("Invalid record in text file '") + inputs[i] + "'");
      cur[i] = (size_t)((nl ? nl + 1 : end) - ((const char*)dbs[i].base + dbs[i].body_off));
    }
    it.pos = dbs[i].pos_of(it.key);
    heap.push(it);
  };
  for(int i = 0; i < n; ++i) push(i);
  const unsigned key_bytes = dbs[0].key_bytes, ocl = ocl_min;
  const uint64_t maxv = ocl >= 8 ? ~(uint64_t)0 : (((uint64_t)1 << (8 * ocl)) - 1);
  uint64_t inter = 0, winter = 0, uni = 0, wuni = 0;
  std::string line;
  while(!heap.empty()) {
    item top = heap.top();
    uint64_t sum = 0, minc = std::numeric_limits<uint64_t>::max(), maxc = 0;
    int present = 0;
    while(!heap.empty() && mer_equal(heap.top().key, top.key)) {
      const int i = heap.top().src;
      const uint64_t v = heap.top().val;
      heap.pop();
      sum += v; minc = std::min(minc, v); maxc = std::max(maxc, v); ++present;
      push(i);
    }
    if(present < n) minc = 0;
    if(op == MERGE_JACCARD) { inter += minc > 0; winter += minc; uni += 1; wuni += maxc; continue; }
    const uint64_t val = op == MERGE_MIN ? minc : op == MERGE_MAX ? maxc : sum;
    if(val >= lower && val <= upper) {
      if(text) {
        line = mer_to_string(top.key, k); line += ' '; line += std::to_string((unsigned long long)val); line += '\n';
        out.write(line.data(), line.size());
      } else {
        out.write((const char*)top.key, key_bytes);
        uint64_t v = std::min(val, maxv);
        out.write((const char*)&v, ocl);
      }
    }
  }
  if(op == MERGE_JACCARD) out << "Jaccard  " << (double)inter / (double)uni << '\n' << "wJaccard " << (double)winter / (double)wuni << '\n';
  out.close();
}

}  // namespace

int main(int argc, char* argv[]) {
  if(argc < 2) { std::cerr << "Too few arguments\nUsage: jellyfish-b200 <cmd> [options] arg...\nWhere <cmd> is one of: count, bc, dump, query, info, histo, stats, merge, inputs.\n"; return 1; }
  std::string cmd = argv[1];
  if(cmd == "count") return count_main(argc - 1, argv + 1);
  if(cmd == "bc") return bc_main(argc - 1, argv + 1);
  if(cmd == "dump")  return dump_main(argc - 1, argv + 1);
  if(cmd == "query") return query_main(argc - 1, argv + 1);
  if(cmd == "info")  return info_main(argc - 1, argv + 1);
  if(cmd == "histo") return histo_main(argc - 1, argv + 1);
  if(cmd == "stats") return stats_main(argc - 1, argv + 1);
  if(cmd == "merge") return merge_main(argc - 1, argv + 1);
  if(cmd == "inputs") return inputs_main(argc - 1, argv + 1);
  if(cmd == "--version" || cmd == "-V") { std::cout << jfgpu_version() << std::endl; return 0; }
  if(cmd == "--help" || cmd == "-h" || cmd == "help") { std::cout << "Usage: jellyfish-b200 <cmd> [options] arg...\nWhere <cmd> is one of: count, bc, dump, query, info, histo, stats, merge.\n"; return 0; }
  std::cerr << "Unknown command '" << cmd << "'\n";
  return 1;
}
