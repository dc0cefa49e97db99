// search_ckpt.cpp — the checkpoint file of a resumable search, on device or host pools.  Layout (version 1), every
// field little-endian and fixed-width, no padding:
//   "TSB200CK"  u32 version  u32 problem  u32 rec
//   i32 a, b, c, m, M, D, pools                               (the call's parameters, search_ckpt.h)
//   u64 tree1, sol1  i64 best1  f64 t_step1, t_step2  u64 steals
//   D times (task order):
//     u64 tree, sol, offloads, parents, launches  i64 best  u32 finished  u32 pools  u64 left  left * rec bytes
//     `pools` times (pool order): i64 best  u64 count  count * rec bytes
//   u64 checksum of every byte before it
// Nothing depends on the GPUs present: D tasks wrap onto them as in the search itself.
#include "search_ckpt.h"

#include <fcntl.h>
#include <sys/stat.h>
#include <unistd.h>

#include <cerrno>
#include <cstdio>
#include <cstring>
#include <string>

#include "tsb200.h"

namespace tsb::ckpt {
namespace {

constexpr char kMagic[8] = {'T', 'S', 'B', '2', '0', '0', 'C', 'K'};
constexpr uint32_t kVersion = 1;

// a word-wise FNV-1a variant: (h ^ w) * P is a bijection of h for every word, so any single changed word changes it
uint64_t checksum(const uint8_t* p, size_t n) {
  uint64_t h = 0xcbf29ce484222325ull;
  size_t i = 0;
  for (; i + 8 <= n; i += 8) {
    uint64_t w = 0;
    for (int k = 0; k < 8; k++) w |= static_cast<uint64_t>(p[i + k]) << (8 * k);
    h = (h ^ w) * 0x100000001b3ull;
  }
  for (; i < n; i++) h = (h ^ p[i]) * 0x100000001b3ull;
  return h ^ (h >> 29);
}

struct Writer {
  std::vector<uint8_t> b;
  void u64(uint64_t v) {
    for (int k = 0; k < 8; k++) b.push_back(static_cast<uint8_t>(v >> (8 * k)));
  }
  void u32(uint32_t v) {
    for (int k = 0; k < 4; k++) b.push_back(static_cast<uint8_t>(v >> (8 * k)));
  }
  void i32(int32_t v) { u32(static_cast<uint32_t>(v)); }
  void i64(int64_t v) { u64(static_cast<uint64_t>(v)); }
  void f64(double v) {
    uint64_t u;
    std::memcpy(&u, &v, 8);
    u64(u);
  }
  void bytes(const std::vector<uint8_t>& v) { b.insert(b.end(), v.begin(), v.end()); }
};

struct Reader {  // every read is bounded; `ok` turns false on the first one past the end
  const uint8_t* p;
  size_t n, at = 0;
  bool ok = true;
  bool take(size_t k) {
    if (!ok || k > n - at) return ok = false;
    return true;
  }
  uint64_t u64() {
    if (!take(8)) return 0;
    uint64_t v = 0;
    for (int k = 0; k < 8; k++) v |= static_cast<uint64_t>(p[at + k]) << (8 * k);
    at += 8;
    return v;
  }
  uint32_t u32() {
    if (!take(4)) return 0;
    uint32_t v = 0;
    for (int k = 0; k < 4; k++) v |= static_cast<uint32_t>(p[at + k]) << (8 * k);
    at += 4;
    return v;
  }
  int32_t i32() { return static_cast<int32_t>(u32()); }
  int64_t i64() { return static_cast<int64_t>(u64()); }
  double f64() {
    const uint64_t u = u64();
    double v;
    std::memcpy(&v, &u, 8);
    return v;
  }
  // `count` records of `rec` bytes
  void records(uint64_t count, uint32_t rec, std::vector<uint8_t>& out) {
    if (!ok || (rec && count > (n - at) / rec)) {
      ok = false;
      return;
    }
    out.assign(p + at, p + at + count * rec);
    at += count * rec;
  }
};

void put_params(Writer& w, const Params& p) {
  w.u32(p.problem);
  w.u32(p.rec);
  for (int32_t v : {p.a, p.b, p.c, p.m, p.M, p.D, p.pools}) w.i32(v);
}

bool write_all(int fd, const uint8_t* p, size_t n) {
  while (n) {
    const ssize_t k = ::write(fd, p, n);
    if (k < 0) return false;
    p += k;
    n -= static_cast<size_t>(k);
  }
  return true;
}

}  // namespace

int save(const char* path, const State& st) {
  Writer w;
  w.b.insert(w.b.end(), kMagic, kMagic + 8);
  w.u32(kVersion);
  put_params(w, st.p);
  w.u64(st.tree1);
  w.u64(st.sol1);
  w.i64(st.best1);
  w.f64(st.t_step1);
  w.f64(st.t_step2);
  w.u64(st.steals);
  const uint32_t rec = st.p.rec;
  for (const TaskState& t : st.tasks) {
    for (uint64_t v : {t.tree, t.sol, t.offloads, t.parents, t.launches}) w.u64(v);
    w.i64(t.best);
    w.u32(t.finished ? 1 : 0);
    w.u32(static_cast<uint32_t>(t.pools.size()));
    w.u64(t.left.size() / rec);
    w.bytes(t.left);
    for (const PoolState& s : t.pools) {
      w.i64(s.best);
      w.u64(s.nodes.size() / rec);
      w.bytes(s.nodes);
    }
  }
  w.u64(checksum(w.b.data(), w.b.size()));

  const std::string tmp = std::string(path) + ".tmp";
  const int fd = ::open(tmp.c_str(), O_WRONLY | O_CREAT | O_TRUNC | O_CLOEXEC, 0644);
  if (fd < 0) return TSB_EINVAL;
  const bool ok = write_all(fd, w.b.data(), w.b.size()) && ::fsync(fd) == 0;
  if (::close(fd) != 0 || !ok || std::rename(tmp.c_str(), path) != 0) {
    ::unlink(tmp.c_str());
    return TSB_EINVAL;
  }
  // the rename itself is durable once the directory is synced
  std::string dir(path);
  const size_t slash = dir.rfind('/');
  dir = slash == std::string::npos ? "." : slash == 0 ? "/" : dir.substr(0, slash);
  if (const int dfd = ::open(dir.c_str(), O_RDONLY | O_DIRECTORY | O_CLOEXEC); dfd >= 0) {
    (void)::fsync(dfd);
    ::close(dfd);
  }
  return TSB_OK;
}

int load(const char* path, const Params& want, State* st) {
  struct stat sb;
  if (::stat(path, &sb) != 0) return errno == ENOENT ? 0 : TSB_EINVAL;
  FILE* f = std::fopen(path, "rb");
  if (!f) return TSB_EINVAL;
  std::vector<uint8_t> buf(static_cast<size_t>(sb.st_size));
  const size_t got = buf.empty() ? 0 : std::fread(buf.data(), 1, buf.size(), f);
  std::fclose(f);
  if (got != buf.size() || buf.size() < 8 + 4 + 8) return TSB_EINVAL;
  const size_t body = buf.size() - 8;
  Reader tail{buf.data() + body, 8};
  if (std::memcmp(buf.data(), kMagic, 8) != 0 || tail.u64() != checksum(buf.data(), body)) return TSB_EINVAL;
  Reader r{buf.data(), body};
  r.at = 8;
  if (r.u32() != kVersion) return TSB_EINVAL;
  Params p;
  p.problem = r.u32();
  p.rec = r.u32();
  for (int32_t* v : {&p.a, &p.b, &p.c, &p.m, &p.M, &p.D, &p.pools}) *v = r.i32();
  if (!r.ok || !(p == want) || p.rec == 0 || p.D < 1 || p.D > 8) return TSB_EINVAL;
  st->p = p;
  st->tree1 = r.u64();
  st->sol1 = r.u64();
  st->best1 = r.i64();
  st->t_step1 = r.f64();
  st->t_step2 = r.f64();
  st->steals = r.u64();
  st->tasks.assign(static_cast<size_t>(p.D), TaskState{});
  for (TaskState& t : st->tasks) {
    for (uint64_t* v : {&t.tree, &t.sol, &t.offloads, &t.parents, &t.launches}) *v = r.u64();
    t.best = r.i64();
    const uint32_t finished = r.u32(), pools = r.u32();
    if (finished > 1 || pools > 4) return TSB_EINVAL;
    if (p.host() && pools != (finished ? 0u : 1u)) return TSB_EINVAL;  // (a host task: its one pool, or its leftovers)
    t.finished = finished == 1;
    r.records(r.u64(), p.rec, t.left);
    t.pools.resize(pools);
    for (PoolState& s : t.pools) {
      s.best = r.i64();
      r.records(r.u64(), p.rec, s.nodes);
    }
  }
  return r.ok && r.at == body ? 1 : TSB_EINVAL;
}

}  // namespace tsb::ckpt
