// jf_sam_input.hpp -- the bytes of a `count --sam` file, as the engine takes them: SAM text, or the inflated BAM stream.
//
// The container is sniffed as htslib's hts_open does: a gzip stream (magic 1f 8b) is inflated first; the bytes are then BAM
// when they start with "BAM\1", else SAM text.  A file starting with "CRAM" is refused: CRAM needs the reference genome and
// its own codecs.  BGZF (gzip members that record their own size in a "BC" extra field, SAM specification 4.1) is inflated on
// a small pool of threads, a group of blocks at a time; any other gzip stream on one thread, member after member.
#ifndef JF_SAM_INPUT_HPP
#define JF_SAM_INPUT_HPP
#include <fcntl.h>
#include <unistd.h>
#include <zlib.h>
#include <algorithm>
#include <cerrno>
#include <cstdint>
#include <cstring>
#include <string>
#include <thread>
#include <vector>

namespace jfb {

// flags of the first chunk of a --sam file (values of JFGPU_FORMAT_SAM / JFGPU_FORMAT_BAM in include/jfgpu.h)
enum : uint32_t { INPUT_FORMAT_SAM = 4u, INPUT_FORMAT_BAM = 8u };

class sam_source {
  enum kind_t { RAW, GZIP, BGZF };
  static constexpr size_t RAW_CHUNK = (size_t)4 << 20;
  static constexpr size_t BGZF_GROUP = 256;                     // blocks inflated side by side (at most 16 MB of output)
  static constexpr size_t BGZF_MAX = (size_t)64 << 10;          // a BGZF block and its output are at most 64 KB
  int fd_ = -1;
  std::string path_;
  kind_t kind_ = RAW;
  std::vector<char> out_; size_t out_pos_ = 0;                  // inflated bytes not handed out yet
  bool eof_ = false;
  std::vector<unsigned char> in_; size_t in_pos_ = 0, in_len_ = 0; bool in_eof_ = false;
  z_stream zs_; bool z_init_ = false, member_open_ = false;
  unsigned threads_ = 1;

  bool read_more(std::string* err) {                            // append file bytes behind in_len_
    if(in_pos_ && in_pos_ == in_len_) in_pos_ = in_len_ = 0;
    if(in_len_ == in_.size()) {                                 // move the unread bytes to the front
      memmove(in_.data(), in_.data() + in_pos_, in_len_ - in_pos_);
      in_len_ -= in_pos_; in_pos_ = 0;
    }
    while(in_len_ < in_.size()) {
      const ssize_t r = ::read(fd_, in_.data() + in_len_, in_.size() - in_len_);
      if(r < 0 && errno == EINTR) continue;
      if(r < 0) { *err = "Error reading SAM file '" + path_ + "': " + strerror(errno); return false; }
      if(r == 0) { in_eof_ = true; break; }
      in_len_ += (size_t)r;
    }
    return true;
  }
  static uint32_t le32(const unsigned char* p) { return p[0] | (uint32_t)p[1] << 8 | (uint32_t)p[2] << 16 | (uint32_t)p[3] << 24; }
  static uint32_t le16(const unsigned char* p) { return p[0] | (uint32_t)p[1] << 8; }
  // total size of the BGZF block whose header is at p (n bytes there), 0 when the header is not a BGZF one
  static size_t bgzf_block_size(const unsigned char* p, size_t n) {
    if(n < 18 || p[0] != 0x1f || p[1] != 0x8b || p[2] != 8 || !(p[3] & 4)) return 0;
    const size_t xlen = le16(p + 10);
    for(size_t q = 12; q + 4 <= 12 + xlen && q + 4 <= n; q += 4 + le16(p + q + 2))
      if(p[q] == 'B' && p[q + 1] == 'C' && le16(p + q + 2) == 2 && q + 6 <= n) return (size_t)le16(p + q + 4) + 1;
    return 0;
  }

  bool refill_bgzf(std::string* err) {
    if(!read_more(err)) return false;
    struct block { size_t at, xlen, size; uint32_t crc, isize; size_t out; };
    std::vector<block> bl;
    size_t pos = in_pos_, total = 0;
    while(bl.size() < BGZF_GROUP && pos < in_len_) {
      const size_t avail = in_len_ - pos;
      if(avail < 18) break;
      const size_t size = bgzf_block_size(in_.data() + pos, avail);
      if(!size) { *err = "Invalid BGZF block in '" + path_ + "': not a BGZF member"; return false; }
      if(size < 26 || size > avail) { if(size < 26) { *err = "Invalid BGZF block size in '" + path_ + "'"; return false; } break; }
      const unsigned char* p = in_.data() + pos;
      block b = { pos, le16(p + 10), size, le32(p + size - 8), le32(p + size - 4), total };
      if(b.isize > BGZF_MAX) { *err = "Invalid BGZF block in '" + path_ + "': more than 64 KB of data"; return false; }
      total += b.isize;
      bl.push_back(b);
      pos += size;
    }
    if(bl.empty()) {
      if(in_pos_ == in_len_ && in_eof_) { eof_ = true; return true; }
      if(in_eof_) { *err = "Truncated BGZF block in '" + path_ + "'"; return false; }
      return true;                                              // (read_more could not fill the header yet)
    }
    out_.resize(total); out_pos_ = 0;
    std::vector<std::string> errs(std::min<size_t>(threads_, bl.size()));
    auto work = [&](size_t t) {
      z_stream z; memset(&z, 0, sizeof(z));
      if(inflateInit2(&z, -15) != Z_OK) { errs[t] = "zlib initialisation failed"; return; }
      for(size_t i = t; i < bl.size(); i += errs.size()) {
        const block& b = bl[i];
        if(!b.isize) { if(b.crc) errs[t] = "Corrupt BGZF block in '" + path_ + "'"; continue; }     // (the end-of-file block)
        inflateReset(&z);
        z.next_in = in_.data() + b.at + 12 + b.xlen; z.avail_in = (uInt)(b.size - 12 - b.xlen - 8);
        z.next_out = (Bytef*)out_.data() + b.out; z.avail_out = b.isize;
        const int r = inflate(&z, Z_FINISH);
        if(r != Z_STREAM_END || z.avail_out != 0 ||
           crc32(0L, (const Bytef*)out_.data() + b.out, b.isize) != b.crc) { errs[t] = "Corrupt BGZF block in '" + path_ + "'"; break; }
      }
      inflateEnd(&z);
    };
    std::vector<std::thread> pool;
    for(size_t t = 1; t < errs.size(); ++t) pool.emplace_back(work, t);
    work(0);
    for(std::thread& th : pool) th.join();
    for(const std::string& e : errs) if(!e.empty()) { *err = e; return false; }
    in_pos_ = pos;
    return true;
  }

  bool refill_gzip(std::string* err) {
    out_.resize(RAW_CHUNK); out_pos_ = 0;
    zs_.next_out = (Bytef*)out_.data(); zs_.avail_out = (uInt)out_.size();
    while(zs_.avail_out) {
      if(in_pos_ == in_len_) {
        if(!in_eof_ && !read_more(err)) return false;
        zs_.next_in = in_.data() + in_pos_; zs_.avail_in = (uInt)(in_len_ - in_pos_);
      }
      if(in_pos_ == in_len_ && in_eof_) {
        if(member_open_) { *err = "Truncated gzip stream in '" + path_ + "'"; return false; }
        eof_ = true; break;
      }
      member_open_ = true;
      const int r = inflate(&zs_, Z_NO_FLUSH);
      in_pos_ = in_len_ - zs_.avail_in;
      if(r == Z_STREAM_END) { member_open_ = false; inflateReset(&zs_); }      // (gzip: further members may follow)
      else if(r != Z_OK && r != Z_BUF_ERROR) { *err = "Corrupt gzip stream in '" + path_ + "'"; return false; }
    }
    out_.resize(out_.size() - zs_.avail_out);
    return true;
  }

  bool refill_raw(std::string* err) {
    out_.resize(RAW_CHUNK); out_pos_ = 0;
    size_t n = 0;
    if(in_pos_ < in_len_) { n = std::min(in_len_ - in_pos_, out_.size()); memcpy(out_.data(), in_.data() + in_pos_, n); in_pos_ += n; }
    while(n < out_.size()) {
      const ssize_t r = ::read(fd_, out_.data() + n, out_.size() - n);
      if(r < 0 && errno == EINTR) continue;
      if(r < 0) { *err = "Error reading SAM file '" + path_ + "': " + strerror(errno); return false; }
      if(r == 0) { eof_ = n == 0; break; }
      n += (size_t)r;
    }
    out_.resize(n);
    return true;
  }

  bool refill(std::string* err) {
    while(out_pos_ == out_.size() && !eof_) {
      out_.clear(); out_pos_ = 0;
      if(!(kind_ == BGZF ? refill_bgzf(err) : kind_ == GZIP ? refill_gzip(err) : refill_raw(err))) return false;
    }
    return true;
  }

 public:
  explicit sam_source(unsigned threads = 0) {
    threads_ = threads ? threads : std::max(1u, std::min(16u, std::thread::hardware_concurrency()));
    memset(&zs_, 0, sizeof(zs_));
  }
  sam_source(const sam_source&) = delete;
  sam_source& operator=(const sam_source&) = delete;
  ~sam_source() { if(z_init_) inflateEnd(&zs_); if(fd_ >= 0) ::close(fd_); }

  // Open and sniff the file; *flags = INPUT_FORMAT_SAM or INPUT_FORMAT_BAM.  "" or the error.
  std::string open(const char* path, uint32_t* flags) {
    path_ = path;
    fd_ = ::open(path, O_RDONLY);
    if(fd_ < 0) return "Can't open SAM file '" + path_ + "'";
    in_.resize(BGZF_GROUP * BGZF_MAX + BGZF_MAX);
    std::string err;
    while(!in_eof_ && in_len_ < 18) if(!read_more(&err)) return err;
    if(in_len_ >= 2 && in_[0] == 0x1f && in_[1] == 0x8b) {
      if(bgzf_block_size(in_.data(), in_len_)) kind_ = BGZF;
      else {
        kind_ = GZIP;
        if(inflateInit2(&zs_, 15 + 16) != Z_OK) return "zlib initialisation failed";
        z_init_ = true;
        zs_.next_in = in_.data(); zs_.avail_in = (uInt)in_len_;
      }
    } else if(in_len_ >= 4 && memcmp(in_.data(), "CRAM", 4) == 0) {
      return "CRAM input is not supported ('" + path_ + "')";
    }
    if(!refill(&err)) return err;
    // sniff the inflated bytes (the first block holds at least the 4 magic bytes of a BAM stream)
    while(out_.size() - out_pos_ < 4 && !eof_) {
      std::vector<char> keep(out_.begin() + out_pos_, out_.end());
      out_.clear(); out_pos_ = 0;
      if(!(kind_ == BGZF ? refill_bgzf(&err) : kind_ == GZIP ? refill_gzip(&err) : refill_raw(&err))) return err;
      out_.insert(out_.begin(), keep.begin(), keep.end());
    }
    const bool bam = out_.size() - out_pos_ >= 4 && memcmp(out_.data() + out_pos_, "BAM\1", 4) == 0;
    *flags = bam ? INPUT_FORMAT_BAM : INPUT_FORMAT_SAM;
    return "";
  }

  // up to n bytes of the (inflated) file; 0 at its end or on an error (*err set)
  size_t read(char* dst, size_t n, std::string* err) {
    size_t got = 0;
    while(got < n) {
      if(!refill(err)) return 0;
      if(out_pos_ == out_.size()) break;
      const size_t t = std::min(n - got, out_.size() - out_pos_);
      memcpy(dst + got, out_.data() + out_pos_, t);
      got += t; out_pos_ += t;
    }
    return got;
  }
};

}  // namespace jfb
#endif
