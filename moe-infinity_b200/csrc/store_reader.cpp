// store_reader.cpp -- the disk tier's reader (SURVEY §8f N3).  Host code only: no CUDA call in this file.
//
// Reads tensors of the reference's on-disk store (`<prefix>/archer_index` + `<prefix>/archer_param_<n>`; format:
// core/aio/archer_tensor_index.cpp:101-132, archer_tensor_handle.cpp:53-86,152-156) into caller-owned (pinned) host memory.
// What it replaces in the reference: ArcherTensorHandle::ReadTensor (archer_tensor_handle.cpp:189-201) ->
// ArcherPrioAioHandle::Read (archer_prio_aio_handle.cpp:37-70) -> ArcherPrioAioContext::{PrepIocbs,AcceptRequest,Schedule}
// (:123-212): a *synchronous* call that cuts the aligned byte range into 1 MiB preads, runs them on ONE worker thread
// ("only one SSD device") and lets a high-priority request overtake low-priority ones between blocks.
//
// Same contract, different machine: an NVMe array feeding a GPU needs many requests in flight, so
//   * requests are asynchronous (ticket = submit, wait/poll later): the caller overlaps the read of chunk i+1 with the
//     host->device copy of chunk i (api.cu: issue_copy of a store-backed expert);
//   * a pool of worker threads (default 8) takes blocks (default 4 MiB) from two queues, high before low, so an on-demand
//     read still overtakes queued prefetch reads at block granularity -- the reference's priority rule;
//   * a request names a LIST of tensors and a byte range of their concatenation (the expert blob layout `w1|w2|w3`,
//     model_topology.cpp:429-431), so one call fills one staging chunk whatever tensor boundaries it crosses;
//   * blocks whose file offset, length and destination are 4096-aligned (kAioAlignment, archer_prio_aio_handle.h:18) go through
//     an O_DIRECT descriptor, everything else (tails, unaligned destinations, file systems without O_DIRECT such as tmpfs)
//     through a buffered one.  Unlike the reference the read never touches bytes past the tensor's end, so destination
//     buffers need no alignment slack.
// Errors are returned (B2M_EIO with a message), never fatal.
#include <errno.h>
#include <fcntl.h>
#include <stdarg.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include <sys/stat.h>
#include <unistd.h>

#include <atomic>
#include <condition_variable>
#include <deque>
#include <memory>
#include <mutex>
#include <string>
#include <thread>
#include <unordered_map>
#include <vector>

#include "../../include/b2m.h"

namespace {

constexpr uint64_t kAlign = 4096;   // kAioAlignment

struct TensorLoc {
  uint32_t file_id;
  int64_t offset;
  uint64_t size;
};

struct Request {
  std::atomic<int> pending{0};
  std::atomic<int> error{0};   // errno of the first failed block (EIO for a short read)
  bool done = false;           // guarded by b2m_store::tmu
};

struct Block {
  std::shared_ptr<Request> req;
  uint32_t file_id;
  int64_t file_off;
  uint64_t len;
  uint8_t* dst;
};

struct Fds {
  int direct = -1, buffered = -1;
};

}  // namespace

struct b2m_store {
  std::string prefix;
  std::unordered_map<uint32_t, TensorLoc> index;
  uint64_t block_bytes = 4u << 20;
  bool try_direct = true;

  std::mutex fd_mu;
  std::unordered_map<uint32_t, Fds> fds;

  std::mutex mu;   // queues
  std::condition_variable cv;
  std::deque<Block> high, low;
  bool stop = false;
  std::vector<std::thread> workers;

  std::mutex tmu;  // tickets
  std::condition_variable tcv;
  std::unordered_map<uint64_t, std::shared_ptr<Request>> tickets;
  uint64_t next_ticket = 1;

  std::atomic<uint64_t> bytes_read{0}, direct_blocks{0}, buffered_blocks{0}, requests{0};

  std::mutex err_mu;
  char err[512] = {0};
};

namespace {

int sfail(b2m_store* s, int code, const char* fmt, ...) {
  if (s) {
    std::lock_guard<std::mutex> g(s->err_mu);
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(s->err, sizeof s->err, fmt, ap);
    va_end(ap);
  }
  return code;
}

// `ArcherTensorIndex::Deserialize` layout: u32 count, then per tensor u32 id | u32 file_id | i64 offset | u64 nbytes | i64 ndim |
// i64 dims[ndim] | 6 option bytes (little endian, packed)
bool parse_index(const std::vector<uint8_t>& d, std::unordered_map<uint32_t, TensorLoc>* out) {
  size_t pos = 0;
  auto need = [&](size_t n) { return pos + n <= d.size(); };
  if (!need(4)) return false;
  uint32_t count;
  memcpy(&count, d.data(), 4);
  pos = 4;
  for (uint32_t i = 0; i < count; ++i) {
    if (!need(32)) return false;
    uint32_t id, file_id;
    int64_t off, ndim;
    uint64_t size;
    memcpy(&id, d.data() + pos, 4);
    memcpy(&file_id, d.data() + pos + 4, 4);
    memcpy(&off, d.data() + pos + 8, 8);
    memcpy(&size, d.data() + pos + 16, 8);
    memcpy(&ndim, d.data() + pos + 24, 8);
    pos += 32;
    if (ndim < 0 || ndim > 64 || off < 0 || !need((size_t)ndim * 8 + 6)) return false;
    pos += (size_t)ndim * 8 + 6;
    (*out)[id] = TensorLoc{file_id, off, size};
  }
  return true;
}

int open_fds(b2m_store* s, uint32_t file_id, Fds* out) {
  std::lock_guard<std::mutex> g(s->fd_mu);
  auto it = s->fds.find(file_id);
  if (it != s->fds.end()) { *out = it->second; return 0; }
  const std::string path = s->prefix + "/archer_param_" + std::to_string(file_id);
  Fds f;
  f.buffered = open(path.c_str(), O_RDONLY | O_CLOEXEC);
  if (f.buffered < 0) return errno ? errno : EIO;
  if (s->try_direct) f.direct = open(path.c_str(), O_RDONLY | O_CLOEXEC | O_DIRECT);   // EINVAL on tmpfs: stay buffered
  s->fds[file_id] = f;
  *out = f;
  return 0;
}

int pread_full(int fd, uint8_t* dst, uint64_t len, int64_t off) {
  uint64_t got = 0;
  while (got < len) {
    const ssize_t n = pread(fd, dst + got, len - got, off + (int64_t)got);
    if (n < 0) {
      if (errno == EINTR) continue;
      return errno ? errno : EIO;
    }
    if (n == 0) return EIO;   // file shorter than its index says
    got += (uint64_t)n;
  }
  return 0;
}

void run_block(b2m_store* s, const Block& b) {
  Fds f;
  int e = open_fds(s, b.file_id, &f);
  if (!e) {
    const bool aligned = f.direct >= 0 && (uint64_t)b.file_off % kAlign == 0 && b.len % kAlign == 0 &&
                         reinterpret_cast<uintptr_t>(b.dst) % kAlign == 0;
    if (aligned) {
      e = pread_full(f.direct, b.dst, b.len, b.file_off);
      if (e == EINVAL) {   // a device with a larger logical block size than 4096
        e = pread_full(f.buffered, b.dst, b.len, b.file_off);
        if (!e) s->buffered_blocks++;
      } else if (!e) {
        s->direct_blocks++;
      }
    } else {
      e = pread_full(f.buffered, b.dst, b.len, b.file_off);
      if (!e) s->buffered_blocks++;
    }
    if (!e) s->bytes_read += b.len;
  }
  if (e) {
    int zero = 0;
    b.req->error.compare_exchange_strong(zero, e);
  }
  if (b.req->pending.fetch_sub(1) == 1) {
    std::lock_guard<std::mutex> g(s->tmu);
    b.req->done = true;
    s->tcv.notify_all();
  }
}

void worker(b2m_store* s) {
  for (;;) {
    Block b;
    {
      std::unique_lock<std::mutex> lk(s->mu);
      s->cv.wait(lk, [&] { return s->stop || !s->high.empty() || !s->low.empty(); });
      if (s->high.empty() && s->low.empty()) return;   // stop, and nothing left to do
      std::deque<Block>& q = !s->high.empty() ? s->high : s->low;
      b = std::move(q.front());
      q.pop_front();
    }
    run_block(s, b);
  }
}

}  // namespace

extern "C" {

int b2m_store_open(const char* prefix, int num_threads, int block_bytes, int flags, b2m_store** out) {
  if (!prefix || !out) return B2M_EINVAL;
  *out = nullptr;
  std::unique_ptr<b2m_store> s(new b2m_store);
  s->prefix = prefix;
  if (block_bytes > 0) s->block_bytes = ((uint64_t)block_bytes + kAlign - 1) & ~(kAlign - 1);
  s->try_direct = (flags & B2M_STORE_NO_ODIRECT) == 0;
  const std::string ipath = s->prefix + "/archer_index";
  FILE* fp = fopen(ipath.c_str(), "rb");
  if (!fp) return B2M_EIO;
  std::vector<uint8_t> data;
  uint8_t buf[65536];
  size_t n;
  while ((n = fread(buf, 1, sizeof buf, fp)) > 0) data.insert(data.end(), buf, buf + n);
  fclose(fp);
  if (!parse_index(data, &s->index)) return B2M_EINVAL;
  const int nt = num_threads > 0 ? (num_threads > 64 ? 64 : num_threads) : 8;
  b2m_store* raw = s.release();
  for (int i = 0; i < nt; ++i) raw->workers.emplace_back(worker, raw);
  *out = raw;
  return B2M_OK;
}

int b2m_store_close(b2m_store* s) {
  if (!s) return B2M_EINVAL;
  {
    std::lock_guard<std::mutex> g(s->mu);
    s->stop = true;
  }
  s->cv.notify_all();
  for (auto& t : s->workers) t.join();   // workers drain both queues first: no request is left half served
  for (auto& kv : s->fds) {
    if (kv.second.direct >= 0) close(kv.second.direct);
    if (kv.second.buffered >= 0) close(kv.second.buffered);
  }
  delete s;
  return B2M_OK;
}

const char* b2m_store_last_error(b2m_store* s) { return s ? s->err : "null store"; }

int b2m_store_count(b2m_store* s) { return s ? (int)s->index.size() : B2M_EINVAL; }

int b2m_store_tensor(b2m_store* s, uint32_t id, uint32_t* file_id, int64_t* offset, uint64_t* nbytes) {
  if (!s) return B2M_EINVAL;
  auto it = s->index.find(id);
  if (it == s->index.end()) return sfail(s, B2M_EINVAL, "tensor %u is not in the index", id);
  if (file_id) *file_id = it->second.file_id;
  if (offset) *offset = it->second.offset;
  if (nbytes) *nbytes = it->second.size;
  return B2M_OK;
}

int b2m_store_blob_bytes(b2m_store* s, const uint32_t* ids, int n, uint64_t* total) {
  if (!s || !ids || n < 0 || !total) return B2M_EINVAL;
  uint64_t t = 0;
  for (int i = 0; i < n; ++i) {
    auto it = s->index.find(ids[i]);
    if (it == s->index.end()) return sfail(s, B2M_EINVAL, "tensor %u is not in the index", ids[i]);
    t += it->second.size;
  }
  *total = t;
  return B2M_OK;
}

int b2m_store_read_range_async(b2m_store* s, const uint32_t* ids, int n, uint64_t blob_off, uint64_t len, void* dst,
                               int high_prio, uint64_t* ticket) {
  if (!s || !ids || n < 1 || !dst || !ticket) return B2M_EINVAL;
  uint64_t total = 0;
  int r = b2m_store_blob_bytes(s, ids, n, &total);
  if (r) return r;
  if (blob_off > total || len > total - blob_off) return sfail(s, B2M_EINVAL, "range [%llu, +%llu) exceeds the %llu-byte blob",
                                                             (unsigned long long)blob_off, (unsigned long long)len, (unsigned long long)total);
  auto req = std::make_shared<Request>();
  std::vector<Block> blocks;
  uint64_t t_begin = 0;   // position of tensor i inside the blob
  for (int i = 0; i < n && len > 0; ++i) {
    const TensorLoc& loc = s->index.find(ids[i])->second;
    const uint64_t t_end = t_begin + loc.size;
    const uint64_t a = blob_off > t_begin ? blob_off : t_begin;
    const uint64_t b = blob_off + len < t_end ? blob_off + len : t_end;
    for (uint64_t p = a; p < b;) {
      // cut at multiples of the block size of the FILE offset, so that interior blocks stay O_DIRECT-aligned
      const uint64_t fo = (uint64_t)loc.offset + (p - t_begin);
      uint64_t l = s->block_bytes - fo % s->block_bytes;
      if (l > b - p) l = b - p;
      blocks.push_back(Block{req, loc.file_id, (int64_t)fo, l, static_cast<uint8_t*>(dst) + (p - blob_off)});
      p += l;
    }
    t_begin = t_end;
  }
  uint64_t tk;
  {
    std::lock_guard<std::mutex> g(s->tmu);
    tk = s->next_ticket++;
    req->done = blocks.empty();
    s->tickets[tk] = req;
  }
  req->pending.store((int)blocks.size());
  s->requests++;
  if (!blocks.empty()) {
    std::lock_guard<std::mutex> g(s->mu);
    std::deque<Block>& q = high_prio ? s->high : s->low;
    for (auto& b : blocks) q.push_back(std::move(b));
  }
  s->cv.notify_all();
  *ticket = tk;
  return B2M_OK;
}

int b2m_store_read_async(b2m_store* s, const uint32_t* ids, int n, void* dst, uint64_t dst_bytes, int high_prio, uint64_t* ticket) {
  uint64_t total = 0;
  int r = b2m_store_blob_bytes(s, ids, n, &total);
  if (r) return r;
  if (dst_bytes < total) return sfail(s, B2M_EINVAL, "destination holds %llu bytes, the tensors need %llu",
                                      (unsigned long long)dst_bytes, (unsigned long long)total);
  return b2m_store_read_range_async(s, ids, n, 0, total, dst, high_prio, ticket);
}

int b2m_store_poll(b2m_store* s, uint64_t ticket) {
  if (!s) return B2M_EINVAL;
  std::lock_guard<std::mutex> g(s->tmu);
  auto it = s->tickets.find(ticket);
  if (it == s->tickets.end()) return B2M_EINVAL;
  if (!it->second->done) return 0;
  return it->second->error.load() ? B2M_EIO : 1;
}

int b2m_store_wait(b2m_store* s, uint64_t ticket) {
  if (!s) return B2M_EINVAL;
  std::shared_ptr<Request> req;
  {
    std::unique_lock<std::mutex> lk(s->tmu);
    auto it = s->tickets.find(ticket);
    if (it == s->tickets.end()) return sfail(s, B2M_EINVAL, "unknown (or already waited-for) ticket %llu", (unsigned long long)ticket);
    req = it->second;
    s->tcv.wait(lk, [&] { return req->done; });
    s->tickets.erase(ticket);
  }
  const int e = req->error.load();
  if (e) return sfail(s, B2M_EIO, "read failed: %s", e == EIO ? "short read (file smaller than its index entry) or I/O error" : strerror(e));
  return B2M_OK;
}

int b2m_store_stats(b2m_store* s, uint64_t out4[4]) {
  if (!s || !out4) return B2M_EINVAL;
  out4[0] = s->bytes_read.load();
  out4[1] = s->direct_blocks.load();
  out4[2] = s->buffered_blocks.load();
  out4[3] = s->requests.load();
  return B2M_OK;
}

}  // extern "C"
