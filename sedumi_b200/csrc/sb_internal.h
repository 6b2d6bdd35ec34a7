// sb_internal.h -- shared internals of libsedumi_b200 (context, error handling, buffers).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include <string>
#include <utility>
#include <vector>
#include "sedumi_b200.h"

namespace sb {

struct Context {
  bool inited = false;
  int device = 0;
  int sm_count = 132;                      // H100 SXM; replaced by the device's count in ensure_init()
  cudaStream_t stream = nullptr;
  int64_t launches = 0;
  int64_t h2d_bytes = 0, d2h_bytes = 0;   // bytes moved over PCIe by this library (every cudaMemcpyAsync, counted below)
  bool profiling = false;
  bool capturing = false;                  // between sb200_graph_begin and sb200_graph_end
  // bump arena for per-call scratch (reset at the start of each public entry point)
  std::vector<std::pair<char *, size_t>> arena_chunks;
  size_t arena_cur = 0, arena_off = 0;
};
// Scratch that lives until the next arena_reset(); never freed in between, so kernels
// enqueued on the stream may keep using it.  Returns nullptr on allocation failure.
void *arena_alloc(size_t bytes);
void arena_reset();
template <typename T> inline T *arena(size_t count) { return (T *)arena_alloc(count * sizeof(T)); }
Context &ctx();
void set_error(const char *fmt, ...);
int  ensure_init();

// Every asynchronous copy of this library goes through here so that the host<->device traffic of a plugin call is
// COUNTED, not estimated (sb200_xfer_bytes; bench.py prints these as e2e.h2d/d2h_bytes_per_step).
// Large copies from / to PAGEABLE host memory (what a MEX host hands over) are staged through a ring of pinned buffers
// by a few host threads (context.cu): the driver's own staging of a pageable cudaMemcpyAsync is single-threaded.
cudaError_t staged_copy(void *dst, const void *src, size_t bytes, cudaMemcpyKind kind, cudaStream_t st, bool *handled);
inline cudaError_t counted_memcpy_async(void *dst, const void *src, size_t bytes, cudaMemcpyKind kind, cudaStream_t st) {
  if (kind == cudaMemcpyHostToDevice) ctx().h2d_bytes += (int64_t)bytes;
  else if (kind == cudaMemcpyDeviceToHost) ctx().d2h_bytes += (int64_t)bytes;
  if (bytes >= ((size_t)4 << 20) && (kind == cudaMemcpyHostToDevice || kind == cudaMemcpyDeviceToHost) && !ctx().capturing) {
    bool handled = false;
    const cudaError_t e = staged_copy(dst, src, bytes, kind, st, &handled);
    if (handled) return e;
  }
  return ::cudaMemcpyAsync(dst, src, bytes, kind, st);
}
#define cudaMemcpyAsync(...) sb::counted_memcpy_async(__VA_ARGS__)

#define SB_CUDA(call)                                                                 \
  do {                                                                                \
    cudaError_t _e = (call);                                                          \
    if (_e != cudaSuccess) {                                                          \
      sb::set_error("%s failed at %s:%d: %s", #call, __FILE__, __LINE__,              \
                    cudaGetErrorString(_e));                                          \
      return 1;                                                                       \
    }                                                                                 \
  } while (0)

#define SB_CHECK(cond, ...)                                                           \
  do {                                                                                \
    if (!(cond)) { sb::set_error(__VA_ARGS__); return 1; }                            \
  } while (0)

#define SB_TRY(expr)                                                                  \
  do { int _rc = (expr); if (_rc) return _rc; } while (0)

// Count + check a kernel launch on the library stream (and time it when profiling is on).
void prof_mark(const char *name);
#define SB_LAUNCH_CHECK_N(name)                                                       \
  do {                                                                                \
    sb::ctx().launches++;                                                             \
    if (sb::ctx().profiling) sb::prof_mark(name);                                     \
    cudaError_t _e = cudaGetLastError();                                              \
    if (_e != cudaSuccess) {                                                          \
      sb::set_error("kernel launch failed at %s:%d: %s", __FILE__, __LINE__,          \
                    cudaGetErrorString(_e));                                          \
      return 1;                                                                       \
    }                                                                                 \
  } while (0)

// RAII device buffer (freed on scope exit).
template <typename T>
struct DevBuf {
  T *p = nullptr;
  size_t n = 0;
  DevBuf() {}
  DevBuf(const DevBuf &) = delete;
  DevBuf &operator=(const DevBuf &) = delete;
  ~DevBuf() { release(); }
  void release() { if (p) cudaFree(p); p = nullptr; n = 0; }
  int alloc(size_t count) {
    release();
    n = count;
    if (count == 0) count = 1;
    cudaError_t e = cudaMalloc((void **)&p, count * sizeof(T));
    if (e != cudaSuccess) { set_error("cudaMalloc(%zu B) failed: %s", count * sizeof(T), cudaGetErrorString(e)); p = nullptr; return 1; }
    return 0;
  }
  int upload(const T *h, size_t count) {
    if (alloc(count)) return 1;
    if (count) {
      cudaError_t e = cudaMemcpyAsync(p, h, count * sizeof(T), cudaMemcpyHostToDevice, ctx().stream);
      if (e != cudaSuccess) { set_error("H2D failed: %s", cudaGetErrorString(e)); return 1; }
    }
    return 0;
  }
  int upload(const std::vector<T> &v) { return upload(v.data(), v.size()); }
  int download(T *h, size_t count) const {
    if (!count) return 0;
    cudaError_t e = cudaMemcpyAsync(h, p, count * sizeof(T), cudaMemcpyDeviceToHost, ctx().stream);
    if (e != cudaSuccess) { set_error("D2H failed: %s", cudaGetErrorString(e)); return 1; }
    return 0;
  }
  int zero() {
    if (!n) return 0;
    cudaError_t e = cudaMemsetAsync(p, 0, n * sizeof(T), ctx().stream);
    if (e != cudaSuccess) { set_error("memset failed: %s", cudaGetErrorString(e)); return 1; }
    return 0;
  }
};

// Content hash of a host buffer: 128 bits.  Word `a` comes from four independent multiply-xorshift lanes over
// 32-byte blocks (the dependent multiply chain of a single-lane hash limits it to ~2 GB/s; four lanes run at memory
// speed); word `b` is an independent rotate-add chain over the same blocks with its own finaliser, so two buffers
// are taken for equal only when both 64-bit functions agree (plans and device mirrors are keyed by these values).
// Buffers above 512 KB are hashed in 256 KB chunks by a small pool of host threads (the plugin boundary hashes
// tens of MB per IPM iteration); the result is a function of the bytes only, independent of the number of threads.
struct Hash128 {
  uint64_t a = 0, b = 0;
  bool operator==(const Hash128 &o) const { return a == o.a && b == o.b; }
  bool operator!=(const Hash128 &o) const { return !(*this == o); }
  bool operator<(const Hash128 &o) const { return a != o.a ? a < o.a : b < o.b; }
};
static const Hash128 HASH_SEED{0x9E3779B97F4A7C15ull, 0xD6E8FEB86659FD93ull};
Hash128 hash128(const void *data, size_t bytes, Hash128 seed = HASH_SEED);

inline uint64_t rotl64(uint64_t x, int r) { return (x << r) | (x >> (64 - r)); }
inline Hash128 hash128_st(const void *data, size_t bytes, Hash128 seed = HASH_SEED) {
  const unsigned char *p = (const unsigned char *)data;
  const uint64_t M = 0xFF51AFD7ED558CCDull;
  uint64_t a = seed.a ^ bytes, b = seed.a * 3, c = seed.a * 5, d = seed.a * 7;
  uint64_t t = seed.b ^ (bytes * 0x9FB21C651E98DF25ull);
  size_t nblk = bytes / 32;
  const uint64_t *w = (const uint64_t *)p;
  for (size_t i = 0; i < nblk; i++, w += 4) {
    a = (a ^ w[0]) * M; a ^= a >> 32;
    b = (b ^ w[1]) * M; b ^= b >> 32;
    c = (c ^ w[2]) * M; c ^= c >> 32;
    d = (d ^ w[3]) * M; d ^= d >> 32;
    t = rotl64(t, 7) + (w[0] ^ rotl64(w[1], 13) ^ rotl64(w[2], 29) ^ rotl64(w[3], 43));
  }
  uint64_t h = a ^ (b * 0xC4CEB9FE1A85EC53ull) ^ (c << 1) ^ (d * M);
  for (size_t i = nblk * 32; i < bytes; i++) { h ^= p[i]; h *= 1099511628211ull; t = rotl64(t, 9) + p[i]; }
  h ^= h >> 33; h *= M; h ^= h >> 33;
  t ^= t >> 31; t *= 0xC4CEB9FE1A85EC53ull; t ^= t >> 29; t *= M; t ^= t >> 32;
  return Hash128{h, t};
}

// ---- device mirrors of host arrays, keyed by content (SURVEY 7.4(4)): a host entry asks for the
// device copy of an input; if an array with the same size and hash is already resident (typically
// the output of the previous plugin call: ADA travelling getada1 -> 2 -> 3 -> blkchol, or L.L used by
// eight solves) the upload is skipped.  Semantically invisible: same bytes in, same result out.
struct MirrorSlot { Hash128 hash; size_t bytes = 0, cap = 0; void *dev = nullptr; uint64_t stamp = 0; int tag = 0; };
// Returns the device copy of (host, bytes); *hit tells whether an upload was avoided.
void *mirror_input(const void *host, size_t bytes, Hash128 *hash_out = nullptr, bool *hit = nullptr);
// A device buffer (persistent slot) to write an output into; after the D2H copy call
// mirror_publish(slot_dev, host, bytes) so that the next call can find it.
void *mirror_output_slot(size_t bytes);
void mirror_publish(void *slot_dev, const void *host, size_t bytes);

// chained key of several arrays: each call folds the previous value in as the seed
inline Hash128 fnv1a(const void *data, size_t bytes, Hash128 h = HASH_SEED) { return hash128(data, bytes, h); }

inline int to_i32(const sb_idx *src, size_t n, std::vector<int> &dst, const char *what) {
  dst.resize(n);
  for (size_t i = 0; i < n; i++) {
    if (src[i] < 0 || src[i] > 2147483647LL) { set_error("%s[%zu]=%lld out of int32 range", what, i, (long long)src[i]); return 1; }
    dst[i] = (int)src[i];
  }
  return 0;
}

}  // namespace sb
