// Host side of the residency: gather a model's scattered parameter tensors into the page-locked staging image that one
// H2D copy moves (and scatter the results back after the one D2H copy).  A whole MobileNetV2 is ~310 tensors / 14 MB; one
// tensor-library copy call per tensor (or one batched call that still dispatches per tensor) costs several times the PCIe
// transfer itself.  No CUDA call in here.
//
// The caller's thread does the work in 256 KB chunks; a small pool of helper threads, parked on a condition variable,
// takes chunks too WHEN the scheduler runs them in time.  Right after a tensor-library parallel region whose OpenMP
// workers are still spinning, freshly spawned-and-joined threads can make the gather several times SLOWER than one
// thread; with chunk stealing a late helper simply finds nothing left, and nobody waits for it.
#include <algorithm>
#include <condition_variable>
#include <cstring>
#include <mutex>
#include <pthread.h>
#include <thread>
#include <vector>

#include "../../include/dfq_b200.h"

namespace {

constexpr size_t kChunk = 256u << 10;

struct Job {
  char* staging; void* const* ptr; const size_t* off; const size_t* prefix; int n; int dir; size_t total;
};

// copy the bytes [lo, hi) of the concatenation of the segments
void copy_range(const Job& j, size_t lo, size_t hi) {
  int i = (int)(std::upper_bound(j.prefix, j.prefix + j.n + 1, lo) - j.prefix) - 1;
  for (; i < j.n && j.prefix[i] < hi; ++i) {
    const size_t a = std::max(lo, j.prefix[i]) - j.prefix[i];
    const size_t b = std::min(hi, j.prefix[i + 1]) - j.prefix[i];
    if (b <= a) continue;
    char* s = j.staging + j.off[i] + a;
    char* t = (char*)j.ptr[i] + a;
    if (j.dir == 0) std::memcpy(s, t, b - a);
    else std::memcpy(t, s, b - a);
  }
}

struct Pool {
  std::mutex m;
  std::condition_variable wake, finished;
  Job job{};
  long next = 0, nchunks = 0, done = 0;
  int helpers = 0;

  // claim one chunk of the current job (under the lock: the job's tables are only ever read for a claimed chunk, and the
  // caller does not return before every claimed chunk is done)
  bool claim(Job& j, long& idx) {
    if (next >= nchunks) return false;
    idx = next++;
    j = job;
    return true;
  }
  void helper() {
    std::unique_lock<std::mutex> lk(m);
    for (;;) {
      Job j; long idx;
      wake.wait(lk, [&] { return next < nchunks; });
      while (claim(j, idx)) {
        lk.unlock();
        copy_range(j, (size_t)idx * kChunk, std::min(j.total, (size_t)(idx + 1) * kChunk));
        lk.lock();
        if (++done == nchunks) finished.notify_all();
      }
    }
  }
  void ensure(int want) {     // under the lock
    for (; helpers < want; ++helpers) std::thread(&Pool::helper, this).detach();
  }
};

Pool* g_pool = nullptr;
std::mutex* g_one_job = nullptr;     // one job at a time through the shared pool

// A forked child inherits the pool's memory but none of its threads (and possibly a locked mutex): start over there.
void forget_pool_in_child() { g_pool = nullptr; g_one_job = nullptr; }

void ensure_globals() {
  static std::once_flag once;
  std::call_once(once, [] { pthread_atfork(nullptr, nullptr, forget_pool_in_child); });
  static std::mutex init_m;
  std::lock_guard<std::mutex> g(init_m);
  // never destroyed: parked helpers may outlive static destruction at process exit
  if (!g_one_job) g_one_job = new std::mutex();
  if (!g_pool) g_pool = new Pool();
}

}  // namespace

extern "C" int dfq_host_copy_segments(void* staging, void* const* ptr, const size_t* bytes, const size_t* off, int n, int dir,
                                      int threads) {
  if (n < 0 || (n > 0 && (!staging || !ptr || !bytes || !off)) || (dir != 0 && dir != 1)) return DFQ_E_ARG;
  if (n == 0) return DFQ_OK;
  std::vector<size_t> prefix((size_t)n + 1, 0);
  for (int i = 0; i < n; ++i) {
    if (bytes[i] && !ptr[i]) return DFQ_E_ARG;
    prefix[i + 1] = prefix[i] + bytes[i];
  }
  Job j{(char*)staging, ptr, off, prefix.data(), n, dir, prefix[n]};
  if (j.total == 0) return DFQ_OK;
  const long nchunks = (long)((j.total + kChunk - 1) / kChunk);
  int T = threads > 0 ? threads : (int)std::min(4u, std::max(1u, std::thread::hardware_concurrency()));
  T = (int)std::min<long>(T, (nchunks + 3) / 4);        // at least ~1 MB per thread
  if (T <= 1) {
    copy_range(j, 0, j.total);
    return DFQ_OK;
  }
  ensure_globals();
  std::lock_guard<std::mutex> serial(*g_one_job);
  Pool& p = *g_pool;
  std::unique_lock<std::mutex> lk(p.m);
  try { p.ensure(T - 1); } catch (...) { }              // no helper threads available: this thread does every chunk
  p.job = j; p.next = 0; p.nchunks = nchunks; p.done = 0;
  p.wake.notify_all();
  Job mine; long idx;
  while (p.claim(mine, idx)) {
    lk.unlock();
    copy_range(mine, (size_t)idx * kChunk, std::min(mine.total, (size_t)(idx + 1) * kChunk));
    lk.lock();
    ++p.done;
  }
  p.finished.wait(lk, [&] { return p.done == p.nchunks; });
  p.nchunks = 0; p.next = 0;                            // nothing to claim until the next job is posted
  return DFQ_OK;
}
