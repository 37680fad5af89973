// jf_inputs.hpp -- the input side of `count` / `bc` on the host: the sequence files of the command line and the standard
// output of generator commands (-g / -G / -S), turned into one sequence of (chunk of text, FILE_BEGIN/FILE_END flags)
// calls for the engine.
//
// Reference behaviour kept (lib/generator_manager.cc:222-274, include/jellyfish/generator_manager.hpp:113-123,
// sub_commands/count_main.cc:260-267,297-303,337-342, stream_manager.hpp): the command file holds one shell command per
// line, blank lines and lines whose first non-blank character is '#' are skipped; at most G commands run at the same time,
// each under `<shell> -c <command>` (shell = -S, else $SHELL, else /bin/sh) with /dev/null as standard input; the output
// of one command is one input "file" (its format is sniffed from its first byte, no k-mer spans two outputs); a command that
// exits with a non-zero status or is killed by a signal is reported ("Command '...' exited with error status N") and the
// run fails with "Some generator commands failed".
//
// Own design: no manager process and no named pipes.  Every running command writes into an anonymous pipe that a pump
// thread empties into a bounded queue of host blocks, so G decompressors really run side by side while the engine takes
// their outputs one after the other (the engine keeps the parser state of ONE file).
#ifndef JF_INPUTS_HPP
#define JF_INPUTS_HPP
#include <fcntl.h>
#include <signal.h>
#include <spawn.h>
#include <sys/types.h>
#include <sys/wait.h>
#include <unistd.h>
#include <atomic>
#include <cerrno>
#include <chrono>
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <condition_variable>
#include <deque>
#include <fstream>
#include <functional>
#include <memory>
#include <mutex>
#include <queue>
#include <string>
#include <thread>
#include <vector>

#include "jf_sam_input.hpp"

extern char** environ;

namespace jfb {

// flags of a chunk (values of JFGPU_FILE_BEGIN / JFGPU_FILE_END in include/jfgpu.h)
enum : uint32_t { INPUT_FILE_BEGIN = 1u, INPUT_FILE_END = 2u };

struct generator_spec {
  const char* cmds_path = nullptr;     // -g
  uint32_t concurrent = 1;             // -G
  const char* shell = nullptr;         // -S
  bool given() const { return cmds_path != nullptr; }
};

// the commands of a -g file, in order
inline bool read_generator_commands(const char* path, std::vector<std::string>* out, std::string* error) {
  std::ifstream in(path);
  if(!in.good()) { *error = std::string("Failed to open cmds file '") + path + "'"; return false; }
  std::string line;
  while(std::getline(in, line)) {
    const size_t pos = line.find_first_not_of(" \t\n\v\f\r");
    if(pos == std::string::npos || line[pos] == '#') continue;
    out->push_back(line);
  }
  return true;
}

// The process groups of the running commands: SIGTERM / SIGINT / SIGHUP to this process end them too (the reference's manager
// process does the same for its children, generator_manager.cc:120-160), then the signal takes its default course.
namespace detail {
constexpr int MAX_LIVE_GROUPS = 256;
inline std::atomic<pid_t>* live_groups() { static std::atomic<pid_t> g[MAX_LIVE_GROUPS]; return g; }
inline void end_commands_and_reraise(int sig) {
  std::atomic<pid_t>* g = live_groups();
  for(int i = 0; i < MAX_LIVE_GROUPS; ++i) { const pid_t p = g[i].load(); if(p > 0) ::kill(-p, SIGTERM); }
  ::signal(sig, SIG_DFL);
  ::raise(sig);
}
inline void watch_signals_once() {
  static std::once_flag once;
  std::call_once(once, [] {
    struct sigaction act;
    memset(&act, 0, sizeof(act));
    act.sa_handler = end_commands_and_reraise;
    const int sigs[] = { SIGTERM, SIGINT, SIGHUP };
    for(int sg : sigs) {
      struct sigaction old;
      if(sigaction(sg, nullptr, &old) == 0 && old.sa_handler == SIG_DFL) sigaction(sg, &act, nullptr);     // (an ignored signal stays ignored)
    }
  });
}
inline int group_enter(pid_t p) {
  std::atomic<pid_t>* g = live_groups();
  for(int i = 0; i < MAX_LIVE_GROUPS; ++i) { pid_t none = 0; if(g[i].compare_exchange_strong(none, p)) return i; }
  return -1;
}
inline void group_leave(int slot) { if(slot >= 0) live_groups()[slot].store(0); }
}  // namespace detail

// One running generator command: its standard output arrives through read().
class command_stream {
  static constexpr size_t BLOCK = (size_t)4 << 20;      // bytes per read of the pipe
  static constexpr size_t MAX_QUEUED = 64;              // blocks a command may run ahead of the engine (256 MB)
  std::string cmd_;
  pid_t pid_ = -1;
  int fd_ = -1, slot_ = -1;
  std::thread pump_;
  std::mutex mu_;
  std::condition_variable cv_;
  std::deque<std::vector<char>> blocks_;
  size_t head_off_ = 0;
  bool eof_ = false, abandon_ = false;
  std::string error_;

  void pump() {
    while(true) {
      std::vector<char> b(BLOCK);
      size_t n = 0;
      bool end = false;
      while(n < BLOCK) {
        const ssize_t r = ::read(fd_, b.data() + n, BLOCK - n);
        if(r < 0 && errno == EINTR) continue;
        if(r < 0) { std::lock_guard<std::mutex> l(mu_); error_ = std::string("Error reading the output of command '") + cmd_ + "': " + strerror(errno); end = true; break; }
        if(r == 0) { end = true; break; }
        n += (size_t)r;
      }
      b.resize(n);
      std::unique_lock<std::mutex> l(mu_);
      cv_.wait(l, [&] { return blocks_.size() < MAX_QUEUED || abandon_; });
      if(abandon_) return;
      if(n) blocks_.push_back(std::move(b));
      if(end) eof_ = true;
      cv_.notify_all();
      if(end) return;
    }
  }

 public:
  command_stream(const std::string& cmd, const char* shell, std::string* error) : cmd_(cmd) {
    detail::watch_signals_once();
    int pfd[2];
    if(::pipe2(pfd, O_CLOEXEC) != 0) { *error = std::string("Failed to create a pipe for command '") + cmd + "': " + strerror(errno); return; }
    ::fcntl(pfd[0], F_SETPIPE_SZ, 1 << 20);            // (best effort)
    posix_spawn_file_actions_t fa;
    posix_spawn_file_actions_init(&fa);
    posix_spawn_file_actions_addopen(&fa, 0, "/dev/null", O_RDONLY, 0);
    posix_spawn_file_actions_adddup2(&fa, pfd[1], 1);
    char* const argv[] = { const_cast<char*>(shell), const_cast<char*>("-c"), const_cast<char*>(cmd_.c_str()), nullptr };
    posix_spawnattr_t at;                               // own process group: an abandoned command is stopped with what it started
    posix_spawnattr_init(&at);
    posix_spawnattr_setflags(&at, POSIX_SPAWN_SETPGROUP);
    posix_spawnattr_setpgroup(&at, 0);
    const int rc = ::posix_spawn(&pid_, shell, &fa, &at, argv, environ);
    posix_spawnattr_destroy(&at);
    posix_spawn_file_actions_destroy(&fa);
    ::close(pfd[1]);
    if(rc != 0) { pid_ = -1; ::close(pfd[0]); *error = std::string("Failed to run '") + shell + "'. Command '" + cmd + "' not run: " + strerror(rc); return; }
    fd_ = pfd[0];
    slot_ = detail::group_enter(pid_);
    pump_ = std::thread([this] { pump(); });
  }
  command_stream(const command_stream&) = delete;
  command_stream& operator=(const command_stream&) = delete;
  ~command_stream() {
    if(pump_.joinable()) {
      { std::lock_guard<std::mutex> l(mu_); abandon_ = true; cv_.notify_all(); }
      if(pid_ > 0) ::kill(-pid_, SIGTERM);             // (an abandoned command: the run is failing anyway)
      pump_.join();
    }
    if(fd_ >= 0) ::close(fd_);
    if(pid_ > 0) { int st; while(::waitpid(pid_, &st, 0) < 0 && errno == EINTR) {} }
    detail::group_leave(slot_);
  }
  bool started() const { return pid_ > 0; }
  const std::string& command() const { return cmd_; }

  // up to n bytes of the output; 0 = the command closed its output (or the pipe failed: see finish()), or `stop` was raised
  size_t read(char* dst, size_t n, const std::atomic<bool>* stop = nullptr) {
    size_t got = 0;
    std::unique_lock<std::mutex> l(mu_);
    while(got < n) {
      while(blocks_.empty() && !eof_) {
        if(stop && stop->load()) return got;
        cv_.wait_for(l, std::chrono::milliseconds(50));
      }
      if(blocks_.empty()) break;
      std::vector<char>& b = blocks_.front();
      const size_t take = std::min(n - got, b.size() - head_off_);
      memcpy(dst + got, b.data() + head_off_, take);
      got += take; head_off_ += take;
      if(head_off_ == b.size()) { blocks_.pop_front(); head_off_ = 0; cv_.notify_all(); }
    }
    return got;
  }

  // after the output has been read to its end: reap the command; "" or what went wrong (display_status of the reference)
  std::string finish() {
    if(pump_.joinable()) pump_.join();
    if(fd_ >= 0) { ::close(fd_); fd_ = -1; }
    std::string msg;
    { std::lock_guard<std::mutex> l(mu_); msg = error_; }
    if(pid_ > 0) {
      int st = 0;
      pid_t r;
      while((r = ::waitpid(pid_, &st, 0)) < 0 && errno == EINTR) {}
      pid_ = -1;
      detail::group_leave(slot_); slot_ = -1;
      if(r < 0) { if(msg.empty()) msg = std::string("Command '") + cmd_ + "' could not be waited for"; }
      else if(WIFEXITED(st) && WEXITSTATUS(st) != 0) msg = std::string("Command '") + cmd_ + "' exited with error status " + std::to_string(WEXITSTATUS(st));
      else if(WIFSIGNALED(st)) msg = std::string("Command '") + cmd_ + "' killed by signal " + std::to_string(WTERMSIG(st));
    }
    return msg;
  }
};

struct input_buffers {                                   // where the chunks live (pinned host memory for the engine)
  std::function<void*(size_t)> alloc;
  std::function<void(void*)> release;
};

// Files first, then the generator outputs, then the --sam files (stream_manager.hpp:134-145), through `feed(data, n, flags)`
// (non-zero return = stop, its message via feed_error).  The first chunk of a --sam file carries INPUT_FORMAT_SAM or
// INPUT_FORMAT_BAM (jf_sam_input.hpp).  A reader thread fills three buffers ahead of the feeding thread.  Returns "" or the
// error of the run.
inline std::string stream_inputs(const std::vector<const char*>& files, const generator_spec& gen, const input_buffers& mem,
                                 const std::function<int(const char*, size_t, uint32_t)>& feed,
                                 const std::function<std::string()>& feed_error, size_t buf_bytes = (size_t)64 << 20,
                                 const std::vector<const char*>& sam_files = {}) {
  std::vector<std::string> cmds;
  const char* shell = gen.shell;
  if(gen.given()) {
    std::string err;
    if(!read_generator_commands(gen.cmds_path, &cmds, &err)) return err;
    if(!shell) shell = getenv("SHELL");
    if(!shell) shell = "/bin/sh";
  }
  const size_t BUF = buf_bytes;
  struct chunk { char* data; size_t n; uint32_t flags; bool last; std::string error; };
  const int NBUF = 3;
  std::vector<char*> bufs(NBUF);
  for(int i = 0; i < NBUF; ++i) { bufs[i] = (char*)mem.alloc(BUF); if(!bufs[i]) return "pinned host allocation failed"; }
  std::mutex mu; std::condition_variable cv;
  std::queue<chunk> ready; std::queue<char*> freeb;
  for(int i = 0; i < NBUF; ++i) freeb.push(bufs[i]);
  std::atomic<bool> stop(false);                         // the feeding side has failed: read no further, end the commands
  std::thread reader([&] {
    auto get_buf = [&]() { std::unique_lock<std::mutex> l(mu); cv.wait(l, [&] { return !freeb.empty(); }); char* b = freeb.front(); freeb.pop(); return b; };
    auto put = [&](chunk c) { std::unique_lock<std::mutex> l(mu); ready.push(c); cv.notify_all(); };
    // one input, read one chunk ahead so that the last chunk can carry FILE_END; `more(dst, n, &err)` = bytes read, 0 at the end
    auto one_input = [&](const std::function<size_t(char*, size_t, std::string*)>& more, uint32_t begin = INPUT_FILE_BEGIN) -> std::string {
      bool first = true, eof = false;
      std::string io_error;
      auto fill = [&](char* b) -> size_t {
        size_t n = 0;
        while(n < BUF) {
          if(stop.load()) { io_error = "stopped"; eof = true; break; }
          const size_t r = more(b + n, BUF - n, &io_error);
          if(r == 0) { eof = true; break; }                 // (never a silent truncation: a failed read sets io_error)
          n += r;
        }
        return n;
      };
      char* cur = get_buf();
      size_t have = fill(cur);
      while(true) {
        char* nxt = nullptr; size_t nn = 0;
        if(!eof) { nxt = get_buf(); nn = fill(nxt); }
        if(!io_error.empty()) {
          std::unique_lock<std::mutex> l(mu); freeb.push(cur); if(nxt) freeb.push(nxt);
          return io_error;
        }
        const bool last_of_input = eof && nn == 0;
        const uint32_t fl = (first ? begin : 0u) | (last_of_input ? INPUT_FILE_END : 0u);
        put(chunk{cur, have, fl, false, ""});
        first = false;
        if(last_of_input) { if(nxt) { std::unique_lock<std::mutex> l(mu); freeb.push(nxt); } return ""; }
        cur = nxt; have = nn;
      }
    };
    for(size_t fi = 0; fi < files.size() && !stop.load(); ++fi) {
      const int fd = ::open(files[fi], O_RDONLY);
      if(fd < 0) { put(chunk{nullptr, 0, 0, true, std::string("Can't open file '") + files[fi] + "'"}); return; }
      const std::string err = one_input([&](char* dst, size_t n, std::string* e) -> size_t {
        while(true) {
          const ssize_t r = ::read(fd, dst, n);
          if(r < 0 && errno == EINTR) continue;
          if(r < 0) { *e = std::string("Error reading file '") + files[fi] + "': " + strerror(errno); return 0; }
          return (size_t)r;
        }
      });
      ::close(fd);
      if(!err.empty()) { put(chunk{nullptr, 0, 0, true, err}); return; }
    }
    // generator commands: up to `concurrent` of them run at any time; their outputs are taken in the order of the file
    std::deque<std::unique_ptr<command_stream>> running;
    size_t next_cmd = 0;
    const size_t width = std::max<uint32_t>(gen.concurrent, 1);
    std::string failed;
    while(!stop.load() && (next_cmd < cmds.size() || !running.empty())) {
      while(next_cmd < cmds.size() && running.size() < width) {
        std::string err;
        std::unique_ptr<command_stream> cs(new command_stream(cmds[next_cmd], shell, &err));
        ++next_cmd;
        if(!cs->started()) { failed = err; break; }
        running.push_back(std::move(cs));
      }
      if(!failed.empty() || running.empty()) break;
      command_stream& cs = *running.front();
      std::string err = one_input([&](char* dst, size_t n, std::string*) -> size_t { return cs.read(dst, n, &stop); });
      if(err.empty()) err = cs.finish();
      running.pop_front();
      if(!err.empty()) { failed = err; break; }
    }
    running.clear();                                        // (terminates what is still running after a failure)
    if(stop.load()) { put(chunk{nullptr, 0, 0, true, ""}); return; }
    if(!failed.empty()) { put(chunk{nullptr, 0, 0, true, failed + "\nSome generator commands failed"}); return; }
    for(size_t fi = 0; fi < sam_files.size() && !stop.load(); ++fi) {
      sam_source src;
      uint32_t form = 0;
      std::string err = src.open(sam_files[fi], &form);
      if(err.empty()) err = one_input([&](char* dst, size_t n, std::string* e) { return src.read(dst, n, e); }, INPUT_FILE_BEGIN | form);
      if(!err.empty()) { put(chunk{nullptr, 0, 0, true, err}); return; }
    }
    put(chunk{nullptr, 0, 0, true, ""});
  });
  std::string error;
  int feed_rc = 0;
  while(true) {
    chunk ck;
    { std::unique_lock<std::mutex> l(mu); cv.wait(l, [&] { return !ready.empty(); }); ck = ready.front(); ready.pop(); }
    if(ck.last) { if(!ck.error.empty() && error.empty()) error = ck.error; break; }
    if(!feed_rc && error.empty()) {
      feed_rc = feed(ck.data, ck.n, ck.flags);
      if(feed_rc) { error = feed_error(); stop.store(true); }
    }
    { std::unique_lock<std::mutex> l(mu); freeb.push(ck.data); cv.notify_all(); }
  }
  reader.join();
  for(int i = 0; i < NBUF; ++i) mem.release(bufs[i]);
  return error;
}

}  // namespace jfb
#endif
