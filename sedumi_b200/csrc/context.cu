// context.cu -- library context: device selection, stream, error text, raw memory helpers.
#include <stdarg.h>
#include <atomic>
#include <condition_variable>
#include <functional>
#include <string.h>
#include <mutex>
#include <thread>
#include "sb_internal.h"

namespace sb {

static Context g_ctx;
static uint64_t g_mirror_clock = 0;
static uint64_t g_call_stamp = 0;          // mirror slots stamped after this value belong to the current host call
static thread_local char g_err[1024] = "";

Context &ctx() { return g_ctx; }

// ---------------------------------------------------------------- chunked, multi-threaded content hash
// hash128(data) = hash128_st(data)                                   for up to HASH_PAR_MIN bytes
//               = hash128_st(array of hash128_st(chunk_i), seed)     above, chunks of HASH_CHUNK bytes,
// so the value depends on the bytes only.  Workers are created on first use and sleep on a condition variable
// between jobs (after a short spin, so that back-to-back plugin calls do not pay the wake-up).
//
// Job hand-over.  The submitter publishes a job (parameters + generation g) under `mu`; a worker copies the
// parameters under the same mutex and may claim chunk i only by a compare-and-swap on `next` = (g << 32 | i):
// a worker that is late (still holding an older generation) sees a foreign tag, claims nothing and writes nothing.
// Every claimed chunk bumps `done` after its result is stored and the submitter waits for done == nchunks, so no
// write to `out` can be outstanding when the next job resizes it.
static const size_t HASH_PAR_MIN = 512 * 1024, HASH_CHUNK = 256 * 1024;
namespace {
struct HashJob { const unsigned char *data; size_t bytes, nchunks; Hash128 seed; Hash128 *out; uint64_t gen; };
struct HashPool {
  std::vector<std::thread> th;
  std::mutex mu;
  std::condition_variable cv;
  HashJob job{nullptr, 0, 0, HASH_SEED, nullptr, 0};
  std::vector<Hash128> out;
  std::atomic<uint64_t> next{0};           // (generation << 32) | next unclaimed chunk
  std::atomic<size_t> done{0};
  std::atomic<uint64_t> gen{0};
  bool stop = false;
  void work(const HashJob &J) {
    for (;;) {
      uint64_t cur = next.load(std::memory_order_acquire);
      if ((cur >> 32) != (J.gen & 0xffffffffull)) return;          // the counter belongs to another job
      const size_t i = (size_t)(cur & 0xffffffffull);
      if (i >= J.nchunks) return;
      if (!next.compare_exchange_weak(cur, cur + 1, std::memory_order_acq_rel)) continue;
      const size_t off = i * HASH_CHUNK, len = std::min(HASH_CHUNK, J.bytes - off);
      J.out[i] = hash128_st(J.data + off, len, J.seed);
      done.fetch_add(1, std::memory_order_release);
    }
  }
  void loop() {
    uint64_t seen = 0;
    for (;;) {
      bool got = false;                   // spin briefly for the next job, then sleep
      for (int s = 0; s < 20000 && !got; s++) got = gen.load(std::memory_order_acquire) != seen;
      HashJob J;
      {
        std::unique_lock<std::mutex> lk(mu);
        if (!got) cv.wait(lk, [&] { return stop || gen.load() != seen; });
        if (stop) return;
        J = job;                          // a consistent snapshot: jobs are published under `mu`
      }
      seen = J.gen;
      work(J);
    }
  }
  void start() {
    unsigned hc = std::thread::hardware_concurrency();
    int nt = (int)std::min<unsigned>(7, hc > 1 ? hc - 1 : 0);     // + the calling thread; the value never depends on the count
    if (const char *e = getenv("SB200_HASH_THREADS")) nt = std::max(0, std::min(15, atoi(e) - 1));
    for (int i = 0; i < nt; i++) th.emplace_back([this] { loop(); });
  }
  ~HashPool() {
    { std::lock_guard<std::mutex> lk(mu); stop = true; gen.fetch_add(1); }
    cv.notify_all();
    for (auto &t : th) t.join();
  }
};
HashPool *g_pool = nullptr;
std::mutex g_pool_mu;
}  // namespace

Hash128 hash128(const void *data, size_t bytes, Hash128 seed) {
  if (bytes <= HASH_PAR_MIN) return hash128_st(data, bytes, seed);
  std::lock_guard<std::mutex> one(g_pool_mu);          // one job at a time
  if (!g_pool) { g_pool = new HashPool(); g_pool->start(); }
  HashPool &P = *g_pool;
  HashJob J;
  {
    std::lock_guard<std::mutex> lk(P.mu);
    const size_t nchunks = (bytes + HASH_CHUNK - 1) / HASH_CHUNK;
    if (P.out.size() < nchunks) P.out.resize(nchunks);  // the previous job has fully drained (done == nchunks)
    const uint64_t g = P.gen.load() + 1;
    P.job = HashJob{(const unsigned char *)data, bytes, nchunks, seed, P.out.data(), g};
    P.done.store(0);
    P.next.store((g & 0xffffffffull) << 32, std::memory_order_release);
    P.gen.store(g, std::memory_order_release);
    J = P.job;
  }
  P.cv.notify_all();
  P.work(J);                                            // the calling thread takes its share
  while (P.done.load(std::memory_order_acquire) < J.nchunks) { }
  Hash128 s2{seed.a ^ (uint64_t)bytes, seed.b + (uint64_t)bytes};
  return hash128_st(J.out, sizeof(Hash128) * J.nchunks, s2);
}

// ---------------------------------------------------------------- staged copies of pageable host memory
// H2D: host threads copy chunks of the source into pinned slots (two sets of slots: the DMA of one set overlaps the host
// copies into the other), each slot goes to the device with an asynchronous copy on the caller's stream.  The call returns
// when the source has been read completely (the semantics of cudaMemcpyAsync on pageable memory).
// D2H: the DMAs of one set are enqueued, the previous set is drained to the destination by the host threads; the call
// returns when the destination is complete (again what the pageable call does).
namespace {
struct CopyPool {            // plain mutex / condition-variable fork-join: jobs are 2 MB memcpy's
  std::vector<std::thread> th;
  std::mutex mu;
  std::condition_variable cv_job, cv_done;
  const std::function<void(size_t)> *fn = nullptr;
  size_t n = 0, next = 0, done = 0;
  uint64_t gen = 0;
  bool stop = false;
  void loop() {
    uint64_t seen = 0;
    std::unique_lock<std::mutex> lk(mu);
    for (;;) {
      cv_job.wait(lk, [&] { return stop || gen != seen; });
      if (stop) return;
      seen = gen;
      while (next < n) {
        const size_t i = next++;
        const std::function<void(size_t)> *f = fn;
        lk.unlock();
        (*f)(i);
        lk.lock();
        if (++done == n) cv_done.notify_all();
      }
    }
  }
  void run(size_t count, const std::function<void(size_t)> &f) {      // the caller takes its share; returns when all are done
    std::unique_lock<std::mutex> lk(mu);
    fn = &f; n = count; next = 0; done = 0; gen++;
    cv_job.notify_all();
    while (next < n) {
      const size_t i = next++;
      lk.unlock();
      f(i);
      lk.lock();
      ++done;
    }
    cv_done.wait(lk, [&] { return done == n; });
    n = 0; next = 0;                                                   // late wake-ups find nothing to claim
  }
  void start() {
    unsigned hc = std::thread::hardware_concurrency();
    int nt = (int)std::min<unsigned>(7, hc > 1 ? hc - 1 : 0);
    if (const char *e = getenv("SB200_COPY_THREADS")) nt = std::max(0, std::min(31, atoi(e) - 1));
    for (int i = 0; i < nt; i++) th.emplace_back([this] { loop(); });
  }
  ~CopyPool() {
    { std::lock_guard<std::mutex> lk(mu); stop = true; }
    cv_job.notify_all();
    for (auto &t : th) t.join();
  }
};
const size_t STG_CH = (size_t)2 << 20;     // chunk = pinned slot
const int STG_SLOTS = 8;                   // slots per set, two sets: 32 MB of pinned memory
struct Staging {
  char *pin = nullptr;
  cudaEvent_t ev[2];
  bool pending[2] = {false, false};
  CopyPool pool;
  bool ok = false, tried = false;
  std::mutex mu;                           // one staged copy at a time
};
Staging *g_stg = nullptr;
}  // namespace

cudaError_t staged_copy(void *dst, const void *src, size_t bytes, cudaMemcpyKind kind, cudaStream_t st, bool *handled) {
  *handled = false;
  static const bool off = getenv("SB200_NO_STAGED_COPY") != nullptr;
  if (off) return cudaSuccess;
  const void *host = kind == cudaMemcpyHostToDevice ? src : dst;
  cudaPointerAttributes at;
  if (::cudaPointerGetAttributes(&at, host) != cudaSuccess) { cudaGetLastError(); return cudaSuccess; }
  if (at.type != cudaMemoryTypeUnregistered) return cudaSuccess;      // pinned / managed: the plain asynchronous copy is right
  if (!g_stg) g_stg = new Staging();
  Staging &S = *g_stg;
  std::lock_guard<std::mutex> one(S.mu);
  if (!S.tried) {
    S.tried = true;
    if (::cudaHostAlloc((void **)&S.pin, 2 * STG_SLOTS * STG_CH, cudaHostAllocDefault) == cudaSuccess &&
        cudaEventCreateWithFlags(&S.ev[0], cudaEventDisableTiming) == cudaSuccess &&
        cudaEventCreateWithFlags(&S.ev[1], cudaEventDisableTiming) == cudaSuccess) {
      S.pool.start();
      S.ok = true;
    } else cudaGetLastError();
  }
  if (!S.ok) return cudaSuccess;
  *handled = true;
  cudaError_t e = cudaSuccess;
  for (int s = 0; s < 2; s++)                                          // slots may still feed DMAs of an earlier call
    if (S.pending[s]) { e = cudaEventSynchronize(S.ev[s]); S.pending[s] = false; if (e != cudaSuccess) return e; }
  const size_t nch = (bytes + STG_CH - 1) / STG_CH;
  const size_t nwave = (nch + STG_SLOTS - 1) / STG_SLOTS;
  if (kind == cudaMemcpyHostToDevice) {
    const char *hs = (const char *)src;
    for (size_t w = 0; w < nwave; w++) {
      const int set = (int)(w & 1);
      if (S.pending[set]) { e = cudaEventSynchronize(S.ev[set]); S.pending[set] = false; if (e != cudaSuccess) return e; }
      const size_t c0 = w * STG_SLOTS, cnt = std::min<size_t>(STG_SLOTS, nch - c0);
      char *base = S.pin + (size_t)set * STG_SLOTS * STG_CH;
      const std::function<void(size_t)> f = [&](size_t i) {
        const size_t o = (c0 + i) * STG_CH, len = std::min(STG_CH, bytes - o);
        memcpy(base + i * STG_CH, hs + o, len);
      };
      S.pool.run(cnt, f);
      for (size_t i = 0; i < cnt; i++) {
        const size_t o = (c0 + i) * STG_CH, len = std::min(STG_CH, bytes - o);
        e = (::cudaMemcpyAsync)((char *)dst + o, base + i * STG_CH, len, cudaMemcpyHostToDevice, st);
        if (e != cudaSuccess) return e;
      }
      e = cudaEventRecord(S.ev[set], st);
      if (e != cudaSuccess) return e;
      S.pending[set] = true;
    }
    return cudaSuccess;
  }
  // device -> host
  char *hd = (char *)dst;
  auto drain = [&](size_t w) -> cudaError_t {
    const int set = (int)(w & 1);
    cudaError_t e2 = cudaEventSynchronize(S.ev[set]);
    S.pending[set] = false;
    if (e2 != cudaSuccess) return e2;
    const size_t c0 = w * STG_SLOTS, cnt = std::min<size_t>(STG_SLOTS, nch - c0);
    const char *base = S.pin + (size_t)set * STG_SLOTS * STG_CH;
    const std::function<void(size_t)> f = [&](size_t i) {
      const size_t o = (c0 + i) * STG_CH, len = std::min(STG_CH, bytes - o);
      memcpy(hd + o, base + i * STG_CH, len);
    };
    S.pool.run(cnt, f);
    return cudaSuccess;
  };
  for (size_t w = 0; w < nwave; w++) {
    const int set = (int)(w & 1);
    const size_t c0 = w * STG_SLOTS, cnt = std::min<size_t>(STG_SLOTS, nch - c0);
    char *base = S.pin + (size_t)set * STG_SLOTS * STG_CH;
    for (size_t i = 0; i < cnt; i++) {
      const size_t o = (c0 + i) * STG_CH, len = std::min(STG_CH, bytes - o);
      e = (::cudaMemcpyAsync)(base + i * STG_CH, (const char *)src + o, len, cudaMemcpyDeviceToHost, st);
      if (e != cudaSuccess) return e;
    }
    e = cudaEventRecord(S.ev[set], st);
    if (e != cudaSuccess) return e;
    S.pending[set] = true;
    if (w > 0) { e = drain(w - 1); if (e != cudaSuccess) return e; }
  }
  return drain(nwave - 1);
}

void set_error(const char *fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof g_err, fmt, ap);
  va_end(ap);
}

void arena_reset() {
  Context &c = g_ctx;
  // Work enqueued earlier may still be reading old scratch: drain the stream first.  Calls
  // are coarse (one MEX-level operation each), so this costs nothing measurable.
  if (c.stream && (c.arena_off || c.arena_cur)) cudaStreamSynchronize(c.stream);
  if (c.arena_chunks.size() > 1) {      // coalesce into one chunk big enough for last call
    size_t tot = 0;
    for (auto &ch : c.arena_chunks) { tot += ch.second; cudaFree(ch.first); }
    c.arena_chunks.clear();
    char *p = nullptr;
    if (cudaMalloc((void **)&p, tot) == cudaSuccess) c.arena_chunks.push_back({p, tot});
    else cudaGetLastError();
  }
  c.arena_cur = 0; c.arena_off = 0;
  g_call_stamp = g_mirror_clock;       // mirror slots touched from now on are pinned for this call
}

void *arena_alloc(size_t bytes) {
  Context &c = g_ctx;
  bytes = (bytes + 255) & ~(size_t)255;
  if (bytes == 0) bytes = 256;
  while (c.arena_cur < c.arena_chunks.size()) {
    auto &ch = c.arena_chunks[c.arena_cur];
    if (c.arena_off + bytes <= ch.second) { void *p = ch.first + c.arena_off; c.arena_off += bytes; return p; }
    c.arena_cur++; c.arena_off = 0;
  }
  size_t cap = bytes > ((size_t)64 << 20) ? bytes : ((size_t)64 << 20);
  char *p = nullptr;
  if (cudaMalloc((void **)&p, cap) != cudaSuccess) { cudaGetLastError(); set_error("arena: cudaMalloc(%zu) failed", cap); return nullptr; }
  c.arena_chunks.push_back({p, cap});
  c.arena_cur = c.arena_chunks.size() - 1;
  c.arena_off = bytes;
  return p;
}

// ---- optional per-launch timing: an event after every launch; the interval between consecutive
// events on the (serial) library stream is attributed to the kernel that was just launched.
struct ProfState {
  std::vector<cudaEvent_t> ev;
  std::vector<const char *> names;
  size_t used = 0;
};
static ProfState g_prof;
void prof_mark(const char *name) {
  if (g_prof.used >= g_prof.ev.size()) {
    size_t n = g_prof.ev.size() ? g_prof.ev.size() * 2 : 4096;
    size_t old = g_prof.ev.size();
    g_prof.ev.resize(n);
    for (size_t i = old; i < n; i++) cudaEventCreate(&g_prof.ev[i]);
    g_prof.names.resize(n);
  }
  cudaEventRecord(g_prof.ev[g_prof.used], g_ctx.stream);
  g_prof.names[g_prof.used] = name;
  g_prof.used++;
}

// ---- content-addressed device mirrors
static MirrorSlot g_mirror[12];
static MirrorSlot *mirror_victim(size_t bytes) {
  // 1) least-recently-used slot that is already big enough and not in use by the current call
  MirrorSlot *best = nullptr;
  for (auto &s : g_mirror)
    if (s.dev && s.cap >= bytes && s.stamp <= g_call_stamp && (!best || s.stamp < best->stamp)) best = &s;
  // 2) otherwise an empty slot (one cudaMalloc, paid once), 3) otherwise grow the LRU unprotected slot
  if (!best) for (auto &s : g_mirror) if (!s.dev) { best = &s; break; }
  if (!best) for (auto &s : g_mirror) if (s.stamp <= g_call_stamp && (!best || s.stamp < best->stamp)) best = &s;
  if (!best) { set_error("mirror: no free slot"); return nullptr; }
  if (best->cap < bytes) {
    if (best->dev) cudaFree(best->dev);
    best->dev = nullptr; best->cap = 0;
    size_t cap = (bytes + ((size_t)1 << 20)) & ~(((size_t)1 << 20) - 1);
    if (cudaMalloc(&best->dev, cap) != cudaSuccess) { cudaGetLastError(); set_error("mirror: cudaMalloc(%zu) failed", cap); return nullptr; }
    best->cap = cap;
  }
  best->hash = Hash128{}; best->bytes = 0; best->stamp = ++g_mirror_clock;
  return best;
}
void *mirror_input(const void *host, size_t bytes, Hash128 *hash_out, bool *hit) {
  const Hash128 h = hash128(host, bytes);
  if (hash_out) *hash_out = h;
  for (auto &s : g_mirror)
    if (s.dev && s.bytes == bytes && s.hash == h) { s.stamp = ++g_mirror_clock; if (hit) *hit = true; return s.dev; }
  if (hit) *hit = false;
  MirrorSlot *s = mirror_victim(bytes);
  if (!s) return nullptr;
  if (cudaMemcpyAsync(s->dev, host, bytes, cudaMemcpyHostToDevice, g_ctx.stream) != cudaSuccess) { set_error("mirror: H2D failed"); return nullptr; }
  s->hash = h; s->bytes = bytes;
  return s->dev;
}
void *mirror_output_slot(size_t bytes) {
  MirrorSlot *s = mirror_victim(bytes);
  return s ? s->dev : nullptr;
}
void mirror_publish(void *slot_dev, const void *host, size_t bytes) {
  for (auto &s : g_mirror)
    if (s.dev == slot_dev) { s.hash = hash128(host, bytes); s.bytes = bytes; s.stamp = ++g_mirror_clock; return; }
}

// keeps the stream busy for a few milliseconds so that the host can enqueue a whole iteration behind it: the event
// intervals of the per-kernel profile are then pure device time, free of host launch gaps
__global__ void prof_spin_kernel(long long cycles) {
  const long long t0 = clock64();
  while (clock64() - t0 < cycles) { }
}

int ensure_init() {
  if (g_ctx.inited) return 0;
  return sb200_init(0);
}

}  // namespace sb

extern "C" {

int sb200_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
  return n;
}

int sb200_init(int device) {
  sb::Context &c = sb::ctx();
  if (c.inited && c.device == device) return 0;
  int n = sb200_device_count();
  if (n <= 0) { sb::set_error("sb200_init: no CUDA device visible (the GPU path has no CPU fallback)"); return 1; }
  if (device < 0 || device >= n) { sb::set_error("sb200_init: device %d out of range (%d visible)", device, n); return 1; }
  SB_CUDA(cudaSetDevice(device));
  if (c.stream) { cudaStreamDestroy(c.stream); c.stream = nullptr; }
  SB_CUDA(cudaStreamCreateWithFlags(&c.stream, cudaStreamNonBlocking));
  cudaDeviceProp prop;
  SB_CUDA(cudaGetDeviceProperties(&prop, device));
  c.sm_count = prop.multiProcessorCount;
  c.device = device;
  c.inited = true;
  return 0;
}

void sb200_shutdown(void) {
  sb::Context &c = sb::ctx();
  if (c.stream) cudaStreamDestroy(c.stream);
  c.stream = nullptr;
  c.inited = false;
}

const char *sb200_last_error(void) { return sb::g_err; }

int sb200_sync(void) {
  SB_TRY(sb::ensure_init());
  SB_CUDA(cudaStreamSynchronize(sb::ctx().stream));
  return 0;
}

int sb200_xfer_bytes(int64_t *h2d, int64_t *d2h) {
  if (h2d) *h2d = sb::ctx().h2d_bytes;
  if (d2h) *d2h = sb::ctx().d2h_bytes;
  return 0;
}
void *sb200_stream(void) { return sb::ensure_init() ? nullptr : (void *)sb::ctx().stream; }
int64_t sb200_kernel_launches(void) { return sb::ctx().launches; }

// Profiling: sb200_prof_begin() starts recording (drains the stream first); sb200_prof_end() stops,
// synchronises and writes one line per kernel name into `buf`: "name count total_ms\n".
int sb200_prof_begin(void) {
  SB_TRY(sb::ensure_init());
  SB_CUDA(cudaStreamSynchronize(sb::ctx().stream));
  sb::g_prof.used = 0;
  sb::ctx().profiling = true;
  sb::prof_spin_kernel<<<1, 1, 0, sb::ctx().stream>>>(6000000LL);      // about 3 ms
  sb::prof_mark("__begin__");
  return 0;
}
int sb200_prof_end(char *buf, int64_t buflen) {
  sb::ctx().profiling = false;
  SB_CUDA(cudaStreamSynchronize(sb::ctx().stream));
  std::vector<std::pair<const char *, std::pair<long long, double>>> agg;
  for (size_t i = 1; i < sb::g_prof.used; i++) {
    float ms = 0.f;
    cudaEventElapsedTime(&ms, sb::g_prof.ev[i - 1], sb::g_prof.ev[i]);
    const char *nm = sb::g_prof.names[i];
    size_t j = 0;
    for (; j < agg.size(); j++) if (agg[j].first == nm || !strcmp(agg[j].first, nm)) break;
    if (j == agg.size()) agg.push_back({nm, {0, 0.0}});
    agg[j].second.first++; agg[j].second.second += ms;
  }
  int64_t off = 0;
  if (buflen > 0) buf[0] = 0;
  for (auto &a : agg) {
    int n = snprintf(buf + off, (size_t)(buflen - off), "%s %lld %.6f\n", a.first, a.second.first, a.second.second);
    if (n < 0 || off + n >= buflen) break;
    off += n;
  }
  return 0;
}

// ---- CUDA graphs: record the launches issued on the library stream between begin and end (only the
// *_dev entry points are capture-safe: no allocation, no host copies, no synchronisation), then
// replay them with one launch.  Removes the per-kernel launch latency of the latency-bound iteration.
int sb200_graph_begin(void) {
  SB_TRY(sb::ensure_init());
  SB_CUDA(cudaStreamSynchronize(sb::ctx().stream));
  SB_CUDA(cudaStreamBeginCapture(sb::ctx().stream, cudaStreamCaptureModeThreadLocal));
  sb::ctx().capturing = true;
  return 0;
}
int sb200_graph_end(void **graph_exec) {
  cudaGraph_t g = nullptr;
  sb::ctx().capturing = false;
  SB_CUDA(cudaStreamEndCapture(sb::ctx().stream, &g));
  cudaGraphExec_t ge = nullptr;
  cudaError_t e = cudaGraphInstantiate(&ge, g, 0);
  cudaGraphDestroy(g);
  if (e != cudaSuccess) { sb::set_error("cudaGraphInstantiate failed: %s", cudaGetErrorString(e)); return 1; }
  *graph_exec = (void *)ge;
  return 0;
}
int sb200_graph_launch(void *graph_exec) {
  SB_CUDA(cudaGraphLaunch((cudaGraphExec_t)graph_exec, sb::ctx().stream));
  return 0;
}
int sb200_graph_destroy(void *graph_exec) {
  SB_CUDA(cudaGraphExecDestroy((cudaGraphExec_t)graph_exec));
  return 0;
}

int sb200_dev_alloc(void **p, int64_t bytes) {
  SB_TRY(sb::ensure_init());
  SB_CUDA(cudaMalloc(p, bytes > 0 ? (size_t)bytes : 1));
  return 0;
}
int sb200_dev_free(void *p) { SB_CUDA(cudaFree(p)); return 0; }
// Diagnostics / tests: the 128-bit content key the caches use for `bytes` bytes at `data` (host only, no device needed).
int sb200_content_hash(const void *data, int64_t bytes, uint64_t out[2]) {
  const sb::Hash128 h = sb::hash128(data, (size_t)bytes);
  out[0] = h.a; out[1] = h.b;
  return 0;
}
int sb200_h2d(void *dst, const void *src, int64_t bytes) {
  SB_TRY(sb::ensure_init());
  SB_CUDA(cudaMemcpyAsync(dst, src, (size_t)bytes, cudaMemcpyHostToDevice, sb::ctx().stream));
  return 0;
}
int sb200_d2h(void *dst, const void *src, int64_t bytes) {
  SB_TRY(sb::ensure_init());
  SB_CUDA(cudaMemcpyAsync(dst, src, (size_t)bytes, cudaMemcpyDeviceToHost, sb::ctx().stream));
  SB_CUDA(cudaStreamSynchronize(sb::ctx().stream));
  return 0;
}

}  // extern "C"
