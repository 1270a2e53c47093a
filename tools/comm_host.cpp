// Host-staged communicator: the eleven comm_* functions of engine.hpp without NCCL, for tests that run several ranks
// as processes on ONE device.  Every collective synchronises the stream, copies the send buffer to the host, publishes
// it as the file <dir>/<session>.<seq>.<rank> (written under a temporary name and renamed into place), waits until
// every rank's file for <seq> exists, combines the files in rank order and copies the result back to the device.
// The directory comes from PQB_COMM_DIR; the session tag is the unique id's bytes, so an earlier run's files never
// match.  A rank that does not reach a collective within PQB_COMM_TIMEOUT_MS (default 60 s) makes the others throw
// PQ_ERR_CUDA "host comm: rank r did not reach collective #seq": ranks that diverge show up as a status, not a hang.
//
// What it does not check: NCCL's stream ordering.  Every call here is synchronous with the host, so a caller that
// reads a result back without synchronising its stream first would pass here and fail under NCCL (the engine
// synchronises after every collective it reads back).  comm_group_begin / end do nothing for the same reason.
//
// Every file starts with what its rank called (all-reduce and op, or all-gather, and the size), so ranks that reach
// different collectives throw instead of combining unrelated bytes; after one failed collective every later call throws
// too (the ranks' sequence numbers no longer match).
//
// Built only into tools/libparseable_b200_hostcomm.so (Makefile), a test build selected with PQB_LIB; the product
// library links comm.cpp.
#include <unistd.h>

#include <algorithm>
#include <cerrno>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <random>
#include <string>
#include <thread>
#include <vector>

#include "engine.hpp"

namespace pqb {

namespace {
std::mutex g_mu;
bool g_active = false;
int g_nranks = 0, g_rank = 0;
uint64_t g_epoch = 0;   // bumped by every comm_init_rank, as in comm.cpp
uint64_t g_seq = 0;     // collectives completed in this session
std::string g_failed;   // why a collective of this session failed
std::string g_dir, g_tag;

std::string file_of(uint64_t seq, int rank) { return g_dir + "/" + g_tag + "." + std::to_string(seq) + "." + std::to_string(rank); }

bool read_file(const std::string& path, std::vector<uint8_t>& out) {
  FILE* f = std::fopen(path.c_str(), "rb");
  if (!f) return false;
  out.clear();
  uint8_t buf[1 << 16];
  size_t n;
  while ((n = std::fread(buf, 1, sizeof(buf), f)) > 0) out.insert(out.end(), buf, buf + n);
  const bool ok = !std::ferror(f);
  std::fclose(f);
  return ok;
}

struct Header { uint64_t what; uint64_t bytes; };   // what: op (0-3) of an all-reduce, 16 for an all-gather

[[noreturn]] void fail(const std::string& why) {
  g_failed = why;
  throw Error(PQ_ERR_CUDA, why);
}

// One collective: publish `mine` under its header, return every rank's bytes in rank order
std::vector<std::vector<uint8_t>> exchange(uint64_t what, const std::vector<uint8_t>& payload) {
  if (!g_active) throw Error(PQ_ERR_INVALID_ARG, "no communicator");
  if (!g_failed.empty()) throw Error(PQ_ERR_CUDA, "host comm: an earlier collective failed (" + g_failed + ")");
  const uint64_t seq = g_seq;
  const Header hd{what, payload.size()};
  std::vector<uint8_t> mine(sizeof(Header) + payload.size());
  std::memcpy(mine.data(), &hd, sizeof(Header));
  if (!payload.empty()) std::memcpy(mine.data() + sizeof(Header), payload.data(), payload.size());
  const std::string own = file_of(seq, g_rank), tmp = own + ".tmp";
  {
    FILE* f = std::fopen(tmp.c_str(), "wb");
    if (!f) throw Error(PQ_ERR_IO, "host comm: cannot write " + tmp + ": " + std::strerror(errno));
    const bool ok = mine.empty() || std::fwrite(mine.data(), 1, mine.size(), f) == mine.size();
    if (std::fclose(f) != 0 || !ok) throw Error(PQ_ERR_IO, "host comm: short write to " + tmp);
    if (std::rename(tmp.c_str(), own.c_str()) != 0) throw Error(PQ_ERR_IO, "host comm: cannot publish " + own + ": " + std::strerror(errno));
  }
  long timeout_ms = 60000;
  if (const char* e = std::getenv("PQB_COMM_TIMEOUT_MS")) timeout_ms = std::strtol(e, nullptr, 10);
  const auto t0 = std::chrono::steady_clock::now();
  std::vector<std::vector<uint8_t>> all(static_cast<size_t>(g_nranks));
  for (int r = 0; r < g_nranks; r++) {
    if (r == g_rank) { all[size_t(r)] = mine; continue; }
    const std::string path = file_of(seq, r);
    // the file appears whole (rename), so existing means complete
    while (access(path.c_str(), F_OK) != 0) {
      if (std::chrono::steady_clock::now() - t0 > std::chrono::milliseconds(timeout_ms))
        fail("host comm: rank " + std::to_string(r) + " did not reach collective #" + std::to_string(seq));
      std::this_thread::sleep_for(std::chrono::microseconds(500));
    }
    if (!read_file(path, all[size_t(r)])) fail("host comm: cannot read " + path);
    Header theirs{~0ull, 0};
    if (all[size_t(r)].size() >= sizeof(Header)) std::memcpy(&theirs, all[size_t(r)].data(), sizeof(Header));
    if (theirs.what != hd.what || theirs.bytes != hd.bytes || all[size_t(r)].size() != mine.size())
      fail("host comm: rank " + std::to_string(r) + " reached a different collective #" + std::to_string(seq) + " (" +
           std::to_string(theirs.what) + ", " + std::to_string(theirs.bytes) + " bytes; this rank " + std::to_string(hd.what) + ", " +
           std::to_string(hd.bytes) + " bytes)");
  }
  for (auto& a : all) a.erase(a.begin(), a.begin() + sizeof(Header));
  // every rank has published <seq>, so every rank has finished reading <seq - 1>
  if (seq) std::remove(file_of(seq - 1, g_rank).c_str());
  g_seq = seq + 1;
  return all;
}

// Copies go on the caller's stream (a non-blocking one) and are waited for: a plain cudaMemcpy runs on the legacy stream,
// which does not order against it, and from pageable memory may return before the device holds the bytes
std::vector<uint8_t> to_host(const void* dev, size_t bytes, cudaStream_t s) {
  std::vector<uint8_t> h(bytes);
  if (bytes) PQB_CUDA(cudaMemcpyAsync(h.data(), dev, bytes, cudaMemcpyDeviceToHost, s));
  PQB_CUDA(cudaStreamSynchronize(s));
  return h;
}

void to_device(void* dev, const std::vector<uint8_t>& h, cudaStream_t s) {
  if (h.empty()) return;
  PQB_CUDA(cudaMemcpyAsync(dev, h.data(), h.size(), cudaMemcpyHostToDevice, s));
  PQB_CUDA(cudaStreamSynchronize(s));
}
}  // namespace

int comm_unique_id(uint8_t* id) {
  std::random_device rd;
  std::memset(id, 0, PQ_COMM_ID_BYTES);
  for (int i = 0; i < 16; i += 4) {
    const uint32_t w = rd() ^ uint32_t(getpid()) * 2654435761u ^ uint32_t(std::chrono::steady_clock::now().time_since_epoch().count());
    std::memcpy(id + i, &w, 4);
  }
  return PQ_OK;
}

int comm_init_rank(const uint8_t* id, int nranks, int rank) {
  std::lock_guard<std::mutex> lk(g_mu);
  if (g_active) throw Error(PQ_ERR_INVALID_ARG, "communicator already initialised");
  if (nranks < 1 || rank < 0 || rank >= nranks) throw Error(PQ_ERR_INVALID_ARG, "bad rank / nranks");
  const char* dir = std::getenv("PQB_COMM_DIR");
  if (!dir || !dir[0]) throw Error(PQ_ERR_INVALID_ARG, "host comm: PQB_COMM_DIR names no exchange directory");
  static const char* const kHex = "0123456789abcdef";
  g_tag.clear();
  for (int i = 0; i < 16; i++) { g_tag += kHex[id[i] >> 4]; g_tag += kHex[id[i] & 15]; }
  g_dir = dir;
  g_nranks = nranks;
  g_rank = rank;
  g_seq = 0;
  g_failed.clear();
  g_epoch++;
  g_active = true;
  return PQ_OK;
}

int comm_destroy() {
  std::lock_guard<std::mutex> lk(g_mu);
  // the last collective's file stays: another rank may not have read it yet
  g_active = false;
  g_nranks = 0;
  return PQ_OK;
}

bool comm_active() { return g_active; }
uint64_t comm_epoch() { return g_epoch; }
void comm_group_begin() {}
void comm_group_end() {}
int comm_nranks() { return g_nranks; }
int comm_rank() { return g_rank; }

void comm_allreduce_u64(void* buf, size_t count, int op, cudaStream_t s) {
  if (!g_active) throw Error(PQ_ERR_INVALID_ARG, "no communicator");
  const auto all = exchange(uint64_t(op), to_host(buf, count * 8, s));
  std::vector<uint64_t> acc(count);
  std::memcpy(acc.data(), all[0].data(), count * 8);
  for (int r = 1; r < g_nranks; r++) {
    const uint8_t* p = all[size_t(r)].data();
    for (size_t i = 0; i < count; i++) {
      uint64_t v;
      std::memcpy(&v, p + i * 8, 8);
      if (op == 0) {
        acc[i] += v;   // wraps in two's complement, as ncclInt64 sum does
      } else if (op == 1 || op == 2) {
        const int64_t a = int64_t(acc[i]), b = int64_t(v);
        acc[i] = uint64_t(op == 1 ? std::min(a, b) : std::max(a, b));
      } else {
        double a, b;
        std::memcpy(&a, &acc[i], 8);
        std::memcpy(&b, &v, 8);
        a += b;   // rank order
        std::memcpy(&acc[i], &a, 8);
      }
    }
  }
  std::vector<uint8_t> out(count * 8);
  if (count) std::memcpy(out.data(), acc.data(), count * 8);
  to_device(buf, out, s);
}

void comm_allgather_bytes(const void* send, void* recv, size_t bytes_per_rank, cudaStream_t s) {
  if (!g_active) throw Error(PQ_ERR_INVALID_ARG, "no communicator");
  const auto all = exchange(16, to_host(send, bytes_per_rank, s));
  std::vector<uint8_t> cat;
  cat.reserve(bytes_per_rank * size_t(g_nranks));
  for (int r = 0; r < g_nranks; r++) cat.insert(cat.end(), all[size_t(r)].begin(), all[size_t(r)].end());
  to_device(recv, cat, s);
}

}  // namespace pqb
