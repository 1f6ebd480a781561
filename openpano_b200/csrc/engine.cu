// engine.cu — context, memory, profiling and the extern "C" entry points of
// libpano_b200.so that are not pure kernel drivers (see include/pano_b200.h).
#include <mutex>
#include "sift.cuh"
#include <pthread.h>
#include <stdarg.h>
#include <time.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <algorithm>

static thread_local std::string g_create_err;

static int ctx_vfail(pano_ctx* ctx, int code, const char* fmt, va_list ap) {
  char buf[512];
  vsnprintf(buf, sizeof(buf), fmt, ap);
  if (ctx) ctx->err = buf; else g_create_err = buf;
  return code;
}

int ctx_fail(pano_ctx* ctx, int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  ctx_vfail(ctx, code, fmt, ap);
  va_end(ap);
  return code;
}

int Sticky::misuse(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  ctx_vfail(ctx, PANO_ERR_INVALID, fmt, ap);
  va_end(ap);
  return fail(PANO_ERR_INVALID);
}

int Sticky::add_check(const char* what, int n, int added, int first, int count, int cap, const void* const* srcs,
                      const int* read, int kind, int fmt, SrcKind* sk) {
  if (err) return err;
  if (finished) return misuse("%s: add after finish", what);
  if (first != added || count <= 0 || count > n - first)
    return misuse("%s: images [%d, %d) added, %d of %d so far", what, first, first + count, added, n);
  if (count > cap) return misuse("%s: %d images in one add (limit %d)", what, count, cap);
  if (!srcs) return misuse("%s: null source list", what);
  for (int k = 0; k < count; ++k)
    if (!srcs[k] && (!read || read[first + k] >= 0)) return misuse("%s: image %d has no source", what, first + k);
  if (int rc = src_kind(ctx, what, kind, sk)) return fail(rc);
  for (int k = 0; k < count; ++k)   // the alignment of the images read only
    if (int rc = src_check(ctx, what, *sk, first + k, fmt, !read || read[first + k] >= 0 ? srcs[k] : nullptr))
      return fail(rc);
  return PANO_OK;
}

int Sticky::finish_check(const char* what, const void* out, int added, int n) {
  if (err) return err;
  if (!out) return misuse("%s: null output", what);
  if (finished) return misuse("%s: already finished", what);
  if (added != n) return misuse("%s: finish after %d of %d images", what, added, n);
  finished = true;
  return PANO_OK;
}

int pix8_check(pano_ctx* ctx, const char* what, int i, int fmt, const void* d_pix) {
  if (!pix8_bytes(fmt))
    return ctx_fail(ctx, PANO_ERR_INVALID, "%s: image %d has format %#x (PANO_PIX_GREY, _RGB, _RGBA or _RGB_PLANAR)",
                    what, i, fmt);
  if (d_pix && fmt == PANO_PIX_RGBA && (reinterpret_cast<uintptr_t>(d_pix) & 3))
    return ctx_fail(ctx, PANO_ERR_INVALID, "%s: image %d: an RGBA source must be 4-byte aligned", what, i);
  return PANO_OK;
}

int src_kind(pano_ctx* ctx, const char* what, int kind, SrcKind* out) {
  const bool u8 = kind == PANO_SRC_RGB8_DEV || kind == PANO_SRC_RGB8_HOST;
  if (!u8 && kind != PANO_SRC_F32_DEV && kind != PANO_SRC_F32_HOST)
    return ctx_fail(ctx, PANO_ERR_INVALID, "%s: unknown source kind %d", what, kind);
  *out = SrcKind{kind, u8, kind == PANO_SRC_F32_HOST || kind == PANO_SRC_RGB8_HOST};
  return PANO_OK;
}

int src_check(pano_ctx* ctx, const char* what, const SrcKind& k, int i, int fmt, const void* px) {
  if (k.u8 ? !pix8_bytes(fmt) : fmt != 3)
    return ctx_fail(ctx, PANO_ERR_INVALID, "%s: image %d: format %#x for source kind %d", what, i, fmt, k.kind);
  return k.u8 ? pix8_check(ctx, what, i, fmt, k.host ? nullptr : px) : PANO_OK;
}

int ctx_cuda(pano_ctx* ctx, cudaError_t e, const char* what) {
  return ctx_fail(ctx, PANO_ERR_CUDA, "CUDA error %s (%s) at %s", cudaGetErrorName(e), cudaGetErrorString(e), what);
}

double g_trace_slow_ms = [] { const char* e = getenv("PANO_TRACE_SLOW_MS"); return e ? atof(e) : 0.0; }();
double pano_now_ms() {
  timespec ts; clock_gettime(CLOCK_MONOTONIC, &ts);
  return ts.tv_sec * 1e3 + ts.tv_nsec * 1e-6;
}
void pano_trace_slow(const char* what, double ms) {
  fprintf(stderr, "[pano slow call] %-28s %9.1f ms  (thread %lx, at %.3f s)\n", what, ms, (unsigned long)pthread_self(), pano_now_ms() * 1e-3);
}

int ctx_alloc(pano_ctx* ctx, void** p, size_t bytes) {
  SlowCall sc("ctx_alloc");
  *p = nullptr;
  bytes = (bytes + 15) / 16 * 16;      // word-granular helper kernels may touch the padding
  if (bytes == 0) bytes = 16;
  if (ctx->cache_limit) {
    // smallest cached block that fits and wastes at most a quarter (+64 KB for the small ones)
    auto it = ctx->cache.lower_bound(bytes);
    if (it != ctx->cache.end() && it->first <= bytes + bytes / 4 + 65536) {
      *p = it->second.p;
      ctx->live[*p] = it->first;
      ctx->cached_bytes -= it->first;
      ctx->cache.erase(it);
      return PANO_OK;
    }
  }
  cudaError_t e = cudaMallocFromPoolAsync(p, bytes, ctx->pool.get(), ctx->stream);
  if (e != cudaSuccess && (ctx->cached_bytes || ctx->sift_plan)) {   // out of memory with blocks parked here: give them back, retry
    cudaGetLastError();
    ctx->sift_plan.reset();
    ctx_cache_release(ctx, 0);
    e = cudaMallocFromPoolAsync(p, bytes, ctx->pool.get(), ctx->stream);
  }
  if (e != cudaSuccess) return ctx_cuda(ctx, e, "cudaMallocAsync");
  if (ctx->cache_limit) ctx->live[*p] = bytes;
  return PANO_OK;
}

void ctx_cache_release(pano_ctx* ctx, size_t keep_bytes) {
  // oldest blocks first: what has not been asked for again is least likely to be
  while (ctx->cached_bytes > keep_bytes && !ctx->cache.empty()) {
    auto oldest = ctx->cache.begin();
    for (auto it = ctx->cache.begin(); it != ctx->cache.end(); ++it)
      if (it->second.stamp < oldest->second.stamp) oldest = it;
    cudaFreeAsync(oldest->second.p, ctx->stream);
    ctx->cached_bytes -= oldest->first;
    ctx->cache.erase(oldest);
  }
}

void ctx_free(pano_ctx* ctx, void* p) {
  SlowCall sc("ctx_free");
  if (!p) return;
  auto f = ctx->live.find(p);
  if (f == ctx->live.end()) { cudaFreeAsync(p, ctx->stream); return; }
  const size_t size = f->second;
  ctx->live.erase(f);
  if (!ctx->cache_limit || size > ctx->cache_limit) { cudaFreeAsync(p, ctx->stream); return; }
  ctx->cache.emplace(size, pano_ctx::CachedBlock{p, ++ctx->cache_stamp});
  ctx->cached_bytes += size;
  const size_t plan_bytes = ctx->sift_plan ? ctx->sift_plan->bytes : 0;   // the kept SIFT plan shares the budget
  if (ctx->cached_bytes + plan_bytes > ctx->cache_limit) ctx_cache_release(ctx, ctx->cache_limit - std::min(plan_bytes, ctx->cache_limit));
}

static void* staging(PinnedBuf& b, size_t bytes) {
  return b.grow(bytes, std::max(bytes, (size_t)1 << 20), cudaHostAllocDefault) == cudaSuccess ? b.get() : nullptr;
}
void* ctx_pinned(pano_ctx* ctx, size_t bytes) { return staging(ctx->pinned, bytes); }
void* ctx_pinned2(pano_ctx* ctx, size_t bytes) {
  // metadata staging is reused across calls: wait for earlier async copies
  if (ctx->pinned2.get()) cudaStreamSynchronize(ctx->stream);
  return staging(ctx->pinned2, bytes);
}

static inline void cpu_relax(int n) {
  for (int i = 0; i < n; ++i) {
#if defined(__x86_64__)
    __builtin_ia32_pause();
#endif
  }
}

// Long waits (another stream's upload / download): poll the driver, but sparsely.
cudaError_t ctx_spin_event(cudaEvent_t ev) {
  for (;;) {
    cudaError_t e = cudaEventQuery(ev);
    if (e != cudaErrorNotReady) return e;
    cpu_relax(400);
  }
}

__global__ void k_set_flag(volatile unsigned* flag, unsigned seq) {
  *flag = seq;
  __threadfence_system();
}

cudaError_t ctx_signal(pano_ctx* ctx, unsigned* token) {
  SlowCall sc("ctx_signal");
  if (!ctx->flag.get()) {
    cudaError_t e = ctx->flag.grow(64, 64, cudaHostAllocMapped | cudaHostAllocPortable);
    if (e != cudaSuccess) return e;
    memset(ctx->flag.get(), 0, 64);
  }
  const unsigned seq = ++ctx->flag_seq;
  ctx->launches++;
  k_set_flag<<<1, 1, 0, ctx->stream>>>((volatile unsigned*)ctx->flag.get(), seq);
  *token = seq;
  return cudaGetLastError();
}

cudaError_t ctx_wait_signal(pano_ctx* ctx, unsigned token) {
  SlowCall sc("ctx_wait_signal(gpu)");
  const volatile unsigned* flag = (const volatile unsigned*)ctx->flag.get();
  if (!flag) return cudaStreamSynchronize(ctx->stream);
  for (long long spins = 0;; ++spins) {
    if ((int)(*flag - token) >= 0) return cudaSuccess;
    cpu_relax(4);
    if (spins > (1LL << 28)) return cudaStreamSynchronize(ctx->stream);   // seconds: let a device fault surface
  }
}

cudaError_t ctx_spin_stream(pano_ctx* ctx) {
  unsigned token = 0;
  cudaError_t e = ctx_signal(ctx, &token);
  if (e != cudaSuccess) return e;
  return ctx_wait_signal(ctx, token);
}

// ---- copy-engine-free small moves
__global__ void k_copy_u32(uint32_t* __restrict__ dst, const uint32_t* __restrict__ src, size_t n) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) dst[i] = src[i];
}
__global__ void k_zero_u32(uint32_t* __restrict__ dst, size_t n) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) dst[i] = 0u;
}

void* ctx_ring(pano_ctx* ctx, size_t bytes) {
  SlowCall sc("ctx_ring");
  bytes = (bytes + 63) / 64 * 64;
  if (bytes > ctx->ring.cap()) {
    if (ctx->ring.get()) cudaStreamSynchronize(ctx->stream);   // queued kernels may still read the old ring
    if (ctx->ring.grow(bytes, std::max(bytes * 2, (size_t)8 << 20), cudaHostAllocMapped | cudaHostAllocPortable) != cudaSuccess) return nullptr;
    ctx->ring_off = 0;
  }
  if (ctx->ring_off + bytes > ctx->ring.cap()) {   // wrap: everything queued so far must have consumed its slice
    cudaStreamSynchronize(ctx->stream);
    ctx->ring_off = 0;
  }
  void* p = (char*)ctx->ring.get() + ctx->ring_off;
  ctx->ring_off += bytes;
  return p;
}

PinnedBuf ctx_small_pinned_get(pano_ctx* ctx, size_t bytes) {
  for (auto it = ctx->small_pinned.begin(); it != ctx->small_pinned.end(); ++it)
    if (it->cap() >= bytes) {
      PinnedBuf b = std::move(*it);
      ctx->small_pinned.erase(it);
      return b;
    }
  PinnedBuf b;
  const size_t want = std::max<size_t>((bytes + 255) / 256 * 256, 1024);
  b.grow(want, want, cudaHostAllocMapped | cudaHostAllocPortable);
  return b;
}
void ctx_small_pinned_put(pano_ctx* ctx, PinnedBuf&& b) { if (b.get()) ctx->small_pinned.push_back(std::move(b)); }

static unsigned small_grid(size_t words) { return (unsigned)std::min<size_t>(std::max<size_t>((words + 255) / 256, 1), 256); }

int ctx_fetch(pano_ctx* ctx, void* d_dst, const void* h_src, size_t bytes) {
  if (!bytes) return PANO_OK;
  const size_t words = (bytes + 3) / 4;
  PANO_LAUNCH(ctx, "k_copy_u32", k_copy_u32, small_grid(words), 256, 0, (uint32_t*)d_dst, (const uint32_t*)h_src, words);
  return PANO_OK;
}
int ctx_store(pano_ctx* ctx, void* h_dst, const void* d_src, size_t bytes) {
  SlowCall sc("ctx_store");
  if (!bytes) return PANO_OK;
  const size_t words = (bytes + 3) / 4;
  PANO_LAUNCH(ctx, "k_copy_u32", k_copy_u32, small_grid(words), 256, 0, (uint32_t*)h_dst, (const uint32_t*)d_src, words);
  return PANO_OK;
}
int ctx_put(pano_ctx* ctx, void* d_dst, const void* h_src, size_t bytes) {
  SlowCall sc("ctx_put");
  if (!bytes) return PANO_OK;
  if (bytes <= 960 * 4) return ctx_put_many(ctx, 1, &d_dst, &h_src, &bytes);
  void* st = ctx_ring(ctx, bytes + 4);
  if (!st) return ctx_fail(ctx, PANO_ERR_CUDA, "pinned ring allocation failed");
  memcpy(st, h_src, bytes);
  return ctx_fetch(ctx, d_dst, st, bytes);
}
int ctx_zero(pano_ctx* ctx, void* d_dst, size_t bytes) {
  SlowCall sc("ctx_zero");
  if (!bytes) return PANO_OK;
  const size_t words = (bytes + 3) / 4;
  PANO_LAUNCH(ctx, "k_zero_u32", k_zero_u32, small_grid(words), 256, 0, (uint32_t*)d_dst, words);
  return PANO_OK;
}

// Several small moves in ONE launch (segment table passed by value): every launch that
// touches host memory pays a PCIe round trip, which stretches to tens of microseconds
// while image uploads / mosaic downloads keep the link busy.
struct CopySegs {
  uint32_t* dst[CTX_MAX_SEGS];
  const uint32_t* src[CTX_MAX_SEGS];   // nullptr = fill with zeros
  unsigned words[CTX_MAX_SEGS];
};
__global__ void k_copy_segs(CopySegs s) {
  uint32_t* d = s.dst[blockIdx.y];
  const uint32_t* q = s.src[blockIdx.y];
  const unsigned n = s.words[blockIdx.y];
  for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) d[i] = q ? q[i] : 0u;
}

static int launch_segs(pano_ctx* ctx, const CopySegs& segs, int n, size_t max_words) {
  if (!n) return PANO_OK;
  dim3 grid((unsigned)small_grid(max_words), (unsigned)n);
  PANO_LAUNCH(ctx, "k_copy_u32", k_copy_segs, grid, 256, 0, segs);
  return PANO_OK;
}

// Small tables (< 4 KB) travel INSIDE the launch as a by-value kernel parameter, which the
// front end delivers with the launch command, so the kernel never stalls on a PCIe read of
// host memory.  (Larger by-value parameters — CUDA 12.1+ takes up to 32 KB — were measured
// to slow concurrent launches from two host threads down badly; they use the ring.)
template <int WORDS>
struct ParamBlob {
  uint32_t* dst[CTX_MAX_SEGS];
  unsigned off[CTX_MAX_SEGS];     // word offset into data, ~0u = fill with zeros
  unsigned words[CTX_MAX_SEGS];
  uint32_t data[WORDS];
};
template <int WORDS>
__global__ void k_copy_params(const __grid_constant__ ParamBlob<WORDS> b) {
  uint32_t* d = b.dst[blockIdx.y];
  const unsigned off = b.off[blockIdx.y], n = b.words[blockIdx.y];
  for (unsigned i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
    d[i] = off == ~0u ? 0u : b.data[off + i];
}

template <int WORDS>
static int put_many_params(pano_ctx* ctx, int n, void* const* d_dst, const void* const* h_src, const size_t* bytes) {
  static ParamBlob<WORDS> blob;            // staging only: copied into the launch by value (ctx calls are serialised,
  static std::mutex mu;                    // different contexts may race -> lock)
  std::lock_guard<std::mutex> lock(mu);
  int m = 0;
  unsigned used = 0, max_words = 0;
  for (int i = 0; i < n; ++i) {
    if (!bytes[i]) continue;
    const unsigned w = (unsigned)((bytes[i] + 3) / 4);
    blob.dst[m] = (uint32_t*)d_dst[i];
    blob.words[m] = w;
    if (h_src[i]) {
      blob.off[m] = used;
      blob.data[used + w - 1] = 0;
      memcpy(blob.data + used, h_src[i], bytes[i]);
      used += w;
    } else {
      blob.off[m] = ~0u;
    }
    max_words = std::max(max_words, w);
    ++m;
  }
  if (!m) return PANO_OK;
  dim3 grid((unsigned)small_grid(max_words), (unsigned)m);
  PANO_LAUNCH(ctx, "k_copy_params", k_copy_params<WORDS>, grid, 256, 0, blob);
  return PANO_OK;
}

int ctx_put_many(pano_ctx* ctx, int n, void* const* d_dst, const void* const* h_src, const size_t* bytes) {
  SlowCall sc("ctx_put_many");
  if (n > CTX_MAX_SEGS) return ctx_fail(ctx, PANO_ERR_INVALID, "ctx_put_many: %d segments", n);
  {
    size_t words = 0;
    for (int i = 0; i < n; ++i) if (h_src[i]) words += (bytes[i] + 3) / 4;
    if (words <= 960) return put_many_params<960>(ctx, n, d_dst, h_src, bytes);        // 4 KB launch
  }
  size_t total = 0;
  for (int i = 0; i < n; ++i) if (h_src[i]) total += align_up(bytes[i] + 4, 64);
  char* st = total ? (char*)ctx_ring(ctx, total) : nullptr;
  if (total && !st) return ctx_fail(ctx, PANO_ERR_CUDA, "pinned ring allocation failed");
  CopySegs segs;
  int m = 0;
  size_t max_words = 0;
  for (int i = 0; i < n; ++i) {
    if (!bytes[i]) continue;
    segs.dst[m] = (uint32_t*)d_dst[i];
    segs.words[m] = (unsigned)((bytes[i] + 3) / 4);
    if (h_src[i]) {
      memcpy(st, h_src[i], bytes[i]);
      segs.src[m] = (const uint32_t*)st;
      st += align_up(bytes[i] + 4, 64);
    } else {
      segs.src[m] = nullptr;
    }
    max_words = std::max(max_words, (size_t)segs.words[m]);
    ++m;
  }
  return launch_segs(ctx, segs, m, max_words);
}

int ctx_store_many(pano_ctx* ctx, int n, void* const* h_pinned_dst, const void* const* d_src, const size_t* bytes) {
  SlowCall sc("ctx_store_many");
  if (n > CTX_MAX_SEGS) return ctx_fail(ctx, PANO_ERR_INVALID, "ctx_store_many: %d segments", n);
  CopySegs segs;
  int m = 0;
  size_t max_words = 0;
  for (int i = 0; i < n; ++i) {
    if (!bytes[i]) continue;
    segs.dst[m] = (uint32_t*)h_pinned_dst[i];
    segs.src[m] = (const uint32_t*)d_src[i];
    segs.words[m] = (unsigned)((bytes[i] + 3) / 4);
    max_words = std::max(max_words, (size_t)segs.words[m]);
    ++m;
  }
  return launch_segs(ctx, segs, m, max_words);
}

// Many device-to-device block moves in ONE launch (the descriptor exchange moves two blocks per
// image: dozens of cudaMemcpyAsync calls cost more host time than the copies take on the GPU).
struct CopySeg { void* dst; const void* src; unsigned long long bytes; };
// Segments on gridDim.y (at most 65,535; two per image of a featureset): the blocks of a y index take
// every gridDim.y-th segment.
__global__ void k_copy_blocks(const CopySeg* __restrict__ segs, int n_segs) {
  for (int s = blockIdx.y; s < n_segs; s += gridDim.y) {
    const CopySeg sg = segs[s];
    const size_t n16 = sg.bytes >> 4;
    const uint4* s4 = (const uint4*)sg.src;
    uint4* d4 = (uint4*)sg.dst;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n16; i += (size_t)gridDim.x * blockDim.x) d4[i] = s4[i];
    const size_t tail0 = n16 << 4;
    for (size_t i = tail0 + (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < sg.bytes; i += (size_t)gridDim.x * blockDim.x)
      ((unsigned char*)sg.dst)[i] = ((const unsigned char*)sg.src)[i];
  }
}

// dst / src must be 16-byte aligned device pointers (or bytes[i] < 16)
int ctx_copy_blocks(pano_ctx* ctx, int n, void* const* dst, const void* const* src, const size_t* bytes) {
  SlowCall sc("ctx_copy_blocks");
  std::vector<CopySeg> segs;
  size_t mx = 0;
  for (int i = 0; i < n; ++i)
    if (bytes[i]) { segs.push_back(CopySeg{dst[i], src[i], (unsigned long long)bytes[i]}); mx = std::max(mx, bytes[i]); }
  if (segs.empty()) return PANO_OK;
  DevBuf<CopySeg> d_segs;
  if (int rc = d_segs.alloc(ctx, segs.size())) return rc;
  if (int rc = ctx_put(ctx, d_segs, segs.data(), segs.size() * sizeof(CopySeg))) return rc;
  dim3 grid((unsigned)std::min<size_t>(std::max<size_t>(mx / (16 * 256 * 4), 1), 64), grid_y((long long)segs.size()));
  PANO_LAUNCH(ctx, "k_copy_blocks", k_copy_blocks, grid, 256, 0, d_segs, (int)segs.size());
  d_segs.reset();
  return PANO_OK;
}

int UploadRing::upload(pano_ctx* ctx, const char* what, int count, const void* const* srcs, const size_t* bytes,
                       const void** d_src, int* slot_out) {
  if (!copy) {
    cudaError_t e = make_stream(&copy);
    for (int b = 0; b < 2 && e == cudaSuccess; ++b) {
      e = make_event(&ev_copied[b], cudaEventDisableTiming);
      if (e == cudaSuccess) e = make_event(&ev_done[b], cudaEventDisableTiming);
    }
    if (e != cudaSuccess) return ctx_cuda(ctx, e, (std::string(what) + ": copy stream / events").c_str());
  }
  const int b = windows & 1;
  std::vector<size_t> off(count);
  size_t total = 0;
  bool all_pinned = true;
  for (int k = 0; k < count; ++k) {
    off[k] = total;
    total += align_up(bytes[k], 256);
    all_pinned = all_pinned && host_is_pinned(srcs[k]);
  }
  // slot b and its staging were last used by window - 2: its upload must be over before the host
  // refills the staging buffer (an event never recorded counts as complete)
  PANO_CUDA(ctx, cudaEventSynchronize(ev_copied[b].get()));
  if (slot_cap[b] < total) {
    slot[b].reset(); slot_cap[b] = 0;
    if (int rc = slot[b].alloc(ctx, total)) return rc;
    slot_cap[b] = total;
    PANO_CUDA(ctx, cudaEventRecord(ev_done[b].get(), ctx->stream));   // the block is ours from here on the context stream
  }
  if (!all_pinned) PANO_CUDA(ctx, stage[b].grow(total, total, cudaHostAllocDefault));
  // the copy must not overwrite the slot before window - 2's kernels have read it
  PANO_CUDA(ctx, cudaStreamWaitEvent(copy.get(), ev_done[b].get(), 0));
  unsigned char* st = (unsigned char*)stage[b].get();
  for (int k = 0; k < count; ++k) {
    const void* src = srcs[k];
    if (!host_is_pinned(src)) {               // pageable: staged, the caller may reuse it on return
      memcpy(st + off[k], src, bytes[k]);
      src = st + off[k];
    }
    PANO_CUDA(ctx, cudaMemcpyAsync(slot[b] + off[k], src, bytes[k], cudaMemcpyHostToDevice, copy.get()));
    d_src[k] = slot[b] + off[k];
  }
  PANO_CUDA(ctx, cudaEventRecord(ev_copied[b].get(), copy.get()));
  PANO_CUDA(ctx, cudaStreamWaitEvent(ctx->stream, ev_copied[b].get(), 0));
  ++windows;
  *slot_out = b;
  return PANO_OK;
}

cudaError_t UploadRing::release(pano_ctx* ctx, int b) { return cudaEventRecord(ev_done[b].get(), ctx->stream); }

static EventPtr get_event(pano_ctx* ctx) {
  EventPtr e;
  if (!ctx->event_pool.empty()) { e = std::move(ctx->event_pool.back()); ctx->event_pool.pop_back(); }
  else make_event(&e, cudaEventDefault);
  return e;
}

void ctx_prof_begin(pano_ctx* ctx, const char* name) {
  ProfEvent pe{name, get_event(ctx), get_event(ctx)};
  cudaEventRecord(pe.start.get(), ctx->stream);
  ctx->prof_pending.push_back(std::move(pe));
}

void ctx_prof_end(pano_ctx* ctx) { cudaEventRecord(ctx->prof_pending.back().stop.get(), ctx->stream); }

static void prof_drain(pano_ctx* ctx) {
  if (ctx->prof_pending.empty()) return;
  cudaStreamSynchronize(ctx->stream);
  for (auto& pe : ctx->prof_pending) {
    float ms = 0;
    cudaEventElapsedTime(&ms, pe.start.get(), pe.stop.get());
    auto& acc = ctx->prof_acc[pe.name];
    acc.first += 1; acc.second += ms;
    ctx->event_pool.push_back(std::move(pe.start));
    ctx->event_pool.push_back(std::move(pe.stop));
  }
  ctx->prof_pending.clear();
}

// the DevBuf owners first (ctx_free uses the cache); the other members go after the body, pool and stream last
pano_ctx::~pano_ctx() {
  sift_plan.reset();
  planet_tab.reset();
  ctx_cache_release(this, 0);
  cudaStreamSynchronize(stream);
  prof_drain(this);
}

extern "C" {

void pano_params_default(pano_params* p) {
  // src/config.cfg:2-69
  p->sift_working_size = 800; p->num_octave = 4; p->num_scale = 7;
  p->scale_factor = 1.4142135623f; p->gauss_sigma = 1.4142135623f; p->gauss_window_factor = 6;
  p->judge_extrema_diff_thres = 2e-3f; p->contrast_thres = 4e-2f; p->pre_color_thres = 5e-2f;
  p->edge_ratio = 6.f; p->calc_offset_depth = 4; p->offset_thres = 0.5f; p->ori_radius = 4.5f;
  p->ori_hist_smooth_count = 2; p->desc_hist_scale_factor = 3; p->desc_int_factor = 512;
  p->match_reject_next_ratio = 0.8f; p->focal_length = 37.f; p->ordered_input = 0; p->lazy_read = 1;
  p->multiband = 0; p->max_output_size = 8000;
}

int pano_create(pano_ctx** out, int device, void* cuda_stream) {
  if (!out) return PANO_ERR_INVALID;
  *out = nullptr;
  int ndev = 0;
  cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev == 0)
    return ctx_fail(nullptr, PANO_ERR_NO_DEVICE, "no CUDA device (%s): this engine has no CPU fallback",
                    e != cudaSuccess ? cudaGetErrorString(e) : "device count 0");
  if (device < 0 || device >= ndev) return ctx_fail(nullptr, PANO_ERR_INVALID, "device %d out of range [0,%d)", device, ndev);
  if ((e = cudaSetDevice(device)) != cudaSuccess) return ctx_cuda(nullptr, e, "cudaSetDevice");
  cudaDeviceProp prop;
  if ((e = cudaGetDeviceProperties(&prop, device)) != cudaSuccess) return ctx_cuda(nullptr, e, "cudaGetDeviceProperties");
  if (prop.major != 9 || prop.minor != 0)   // sm_90a code runs on compute capability 9.0 only
    return ctx_fail(nullptr, PANO_ERR_NO_DEVICE, "device %d is sm_%d%d; libpano_b200 is built for sm_90a only", device, prop.major, prop.minor);
  StreamPtr own_stream;   // a caller's stream is borrowed: never destroyed here
  if (!cuda_stream && (e = make_stream(&own_stream)) != cudaSuccess) return ctx_cuda(nullptr, e, "cudaStreamCreate");
  // a private pool that keeps its freed blocks: the same sizes recur every batch
  PoolPtr pool;
  {
    cudaMemPoolProps props;
    memset(&props, 0, sizeof(props));
    props.allocType = cudaMemAllocationTypePinned;
    props.handleTypes = cudaMemHandleTypeNone;
    props.location.type = cudaMemLocationTypeDevice;
    props.location.id = device;
    cudaMemPool_t p = nullptr;
    if ((e = cudaMemPoolCreate(&p, &props)) != cudaSuccess) return ctx_cuda(nullptr, e, "cudaMemPoolCreate");
    pool.reset(p);
    uint64_t thr = UINT64_MAX;
    cudaMemPoolSetAttribute(p, cudaMemPoolAttrReleaseThreshold, &thr);
  }
  pano_ctx* ctx = new pano_ctx;
  ctx->device = device;
  ctx->num_sms = prop.multiProcessorCount;
  ctx->stream = cuda_stream ? (cudaStream_t)cuda_stream : own_stream.get();
  ctx->own_stream = std::move(own_stream);
  ctx->pool = std::move(pool);
  if (const char* e = getenv("PANO_CACHE_MB")) ctx->cache_limit = (size_t)std::max(0LL, atoll(e)) << 20;
  *out = ctx;
  return PANO_OK;
}

int pano_trim(pano_ctx* ctx) {
  if (!ctx) return PANO_ERR_INVALID;
  ctx_enter(ctx);
  ctx->sift_plan.reset();
  ctx_cache_release(ctx, 0);
  return PANO_OK;
}

int pano_mem_high_water(pano_ctx* ctx, size_t* bytes, int reset) {
  if (!ctx || !bytes) return PANO_ERR_INVALID;
  ctx_enter(ctx);
  unsigned long long v = 0;   // cuuint64_t
  PANO_CUDA(ctx, cudaMemPoolGetAttribute(ctx->pool.get(), cudaMemPoolAttrUsedMemHigh, &v));
  *bytes = (size_t)v;
  if (reset) {
    unsigned long long zero = 0;   // the mark restarts at what is in use now
    PANO_CUDA(ctx, cudaMemPoolSetAttribute(ctx->pool.get(), cudaMemPoolAttrUsedMemHigh, &zero));
  }
  return PANO_OK;
}

void pano_destroy(pano_ctx* ctx) {
  ctx_enter(ctx);
  delete ctx;
}

const char* pano_last_error(const pano_ctx* ctx) { return ctx ? ctx->err.c_str() : g_create_err.c_str(); }

int pano_sync(pano_ctx* ctx) {
  ctx_enter(ctx);
  PANO_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return PANO_OK;
}

void* pano_stream(pano_ctx* ctx) {
  ctx_enter(ctx); return (void*)ctx->stream; }

int pano_profile_enable(pano_ctx* ctx, int on) {
  ctx_enter(ctx);
  prof_drain(ctx);
  ctx->profiling = on != 0;
  return PANO_OK;
}

int pano_profile_reset(pano_ctx* ctx) {
  ctx_enter(ctx);
  prof_drain(ctx);
  ctx->prof_acc.clear();
  return PANO_OK;
}

int pano_profile_read(pano_ctx* ctx, int cap, char* names, int* launches, double* total_ms) {
  ctx_enter(ctx);
  prof_drain(ctx);
  int i = 0;
  for (auto& kv : ctx->prof_acc) {
    if (i < cap) {
      strncpy(names + (size_t)i * 64, kv.first.c_str(), 63);
      names[(size_t)i * 64 + 63] = 0;
      launches[i] = kv.second.first;
      total_ms[i] = kv.second.second;
    }
    ++i;
  }
  return i;
}

long long pano_launch_count(const pano_ctx* ctx) {
  ctx_enter(ctx); return ctx->launches; }
int pano_match_last_exact_rows(const pano_ctx* ctx) {
  ctx_enter(ctx); return ctx->last_match_exact_rows; }
int pano_match_last_nominated_rows(const pano_ctx* ctx) {
  ctx_enter(ctx); return ctx->last_match_nominated_rows; }

// ---------------------------------------------------------------- device utilities
int pano_dev_alloc(pano_ctx* ctx, size_t bytes, void** d_ptr) {
  ctx_enter(ctx); return ctx_alloc(ctx, d_ptr, bytes); }
int pano_dev_free(pano_ctx* ctx, void* d_ptr) {
  ctx_enter(ctx); DevBuf<unsigned char>(ctx, (unsigned char*)d_ptr).reset(); return PANO_OK; }
int pano_dev_upload(pano_ctx* ctx, void* d_dst, const void* h_src, size_t bytes) {
  ctx_enter(ctx);
  PANO_CUDA(ctx, cudaMemcpyAsync(d_dst, h_src, bytes, cudaMemcpyHostToDevice, ctx->stream));
  PANO_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return PANO_OK;
}
int pano_dev_download(pano_ctx* ctx, void* h_dst, const void* d_src, size_t bytes) {
  ctx_enter(ctx);
  PANO_CUDA(ctx, cudaMemcpyAsync(h_dst, d_src, bytes, cudaMemcpyDeviceToHost, ctx->stream));
  PANO_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return PANO_OK;
}

int pano_dev_upload_async(pano_ctx* ctx, void* d_dst, const void* h_src, size_t bytes) {
  ctx_enter(ctx);
  PANO_CUDA(ctx, cudaMemcpyAsync(d_dst, h_src, bytes, cudaMemcpyHostToDevice, ctx->stream));
  return PANO_OK;
}
int pano_dev_download_async(pano_ctx* ctx, void* h_dst, const void* d_src, size_t bytes) {
  ctx_enter(ctx);
  PANO_CUDA(ctx, cudaMemcpyAsync(h_dst, d_src, bytes, cudaMemcpyDeviceToHost, ctx->stream));
  return PANO_OK;
}

int pano_host_alloc(size_t bytes, void** h_ptr) {
  if (!h_ptr) return PANO_ERR_INVALID;
  *h_ptr = nullptr;
  return cudaHostAlloc(h_ptr, bytes ? bytes : 16, cudaHostAllocPortable) == cudaSuccess ? PANO_OK : PANO_ERR_CUDA;
}
int pano_host_free(void* h_ptr) { return cudaFreeHost(h_ptr) == cudaSuccess ? PANO_OK : PANO_ERR_CUDA; }

struct pano_event { EventPtr ev; int device; };

int pano_event_create(pano_ctx* ctx, pano_event** out) {
  ctx_enter(ctx);
  if (!ctx || !out) return PANO_ERR_INVALID;
  std::unique_ptr<pano_event> e(new pano_event);
  e->device = ctx->device;
  cudaError_t err = make_event(&e->ev, cudaEventDisableTiming);
  if (err != cudaSuccess) return ctx_cuda(ctx, err, "cudaEventCreate");
  *out = e.release();
  return PANO_OK;
}
int pano_event_record(pano_ctx* ctx, pano_event* ev) {
  ctx_enter(ctx);
  if (!ctx || !ev) return PANO_ERR_INVALID;
  PANO_CUDA(ctx, cudaEventRecord(ev->ev.get(), ctx->stream));
  return PANO_OK;
}
int pano_event_wait(pano_ctx* ctx, pano_event* ev) {
  ctx_enter(ctx);
  if (!ctx || !ev) return PANO_ERR_INVALID;
  PANO_CUDA(ctx, cudaStreamWaitEvent(ctx->stream, ev->ev.get(), 0));
  return PANO_OK;
}
int pano_event_sync(pano_event* ev) {
  if (ev) cudaSetDevice(ev->device);
  if (!ev) return PANO_ERR_INVALID;
  return ctx_spin_event(ev->ev.get()) == cudaSuccess ? PANO_OK : PANO_ERR_CUDA;
}
void pano_event_destroy(pano_event* ev) {
  if (ev) cudaSetDevice(ev->device);
  delete ev;
}

// ---------------------------------------------------------------- features

int ctx_sift_cap(pano_ctx* ctx) {
  if (ctx->sift_cap <= 0) {
    const char* e = getenv("PANO_SIFT_CAP");            // test hook: start small to exercise the growth path
    ctx->sift_cap = e ? std::max(256, atoi(e)) : SIFT_CAP_DEFAULT;
  }
  return ctx->sift_cap;
}

// channels == nullptr: h×w×3 f32 device images; otherwise 8-bit device images in PANO_PIX_* format channels[i]
static int sift_detect_dev(pano_ctx* ctx, int n, const void* const* d_src, const int* channels, const int* w,
                           const int* h, const pano_params* p, pano_featureset** out) {
  std::unique_ptr<pano_featureset> fs(new pano_featureset);
  fs->ctx = ctx;
  // kept for the capacity retry of featureset_sync_counts
  fs->src.assign(d_src, d_src + n); fs->src_w.assign(w, w + n); fs->src_h.assign(h, h + n); fs->src_params = *p;
  if (channels) fs->src_channels.assign(channels, channels + n);
  int rc = sift_run_batch(ctx, n, d_src, channels, w, h, p, fs.get(), nullptr, ctx_sift_cap(ctx));
  if (rc != 0) return rc;
  *out = fs.release();
  return PANO_OK;
}

int pano_sift_detect_batch_dev(pano_ctx* ctx, int n, const float* const* d_rgb, const int* w, const int* h,
                               const pano_params* p, pano_featureset** out) {
  ctx_enter(ctx);
  if (!ctx || !out) return PANO_ERR_INVALID;
  *out = nullptr;
  if (n <= 0 || !d_rgb || !w || !h || !p) return ctx_fail(ctx, PANO_ERR_INVALID, "sift: bad argument");
  return sift_detect_dev(ctx, n, (const void* const*)d_rgb, nullptr, w, h, p, out);
}

bool host_is_pinned(const void* p) {
  cudaPointerAttributes a;
  if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return false; }
  return a.type == cudaMemoryTypeHost;
}

// Uploads host images through one pinned staging buffer (async H2D on the ctx
// stream), then runs the device path.  channels == nullptr: h×w×3 f32 images; otherwise
// 8-bit images in format channels[i].  Every image starts on a 256-byte boundary of d_block (so RGBA taps
// are aligned).
static int upload_images(pano_ctx* ctx, int n, const void* const* src, const int* channels, const int* w, const int* h,
                         std::vector<const void*>& d_imgs, DevBuf<unsigned char>& d_block) {
  size_t total = 0;
  std::vector<size_t> offs(n), bytes(n);
  for (int i = 0; i < n; ++i) {
    if (!src[i] || w[i] <= 0 || h[i] <= 0) return ctx_fail(ctx, PANO_ERR_INVALID, "image %d: null or empty", i);
    offs[i] = total;
    bytes[i] = src_bytes(w[i], h[i], channels, channels ? channels[i] : 3);
    total += align_up(bytes[i], 256);
  }
  if (int rc = d_block.alloc(ctx, total)) return rc;
  // the staging buffer may still feed an earlier async copy
  PANO_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  bool all_pinned = true;
  for (int i = 0; i < n; ++i) all_pinned = all_pinned && host_is_pinned(src[i]);
  unsigned char* st = all_pinned ? (unsigned char*)ctx_pinned(ctx, 64) : (unsigned char*)ctx_pinned(ctx, total);
  if (!st) return ctx_fail(ctx, PANO_ERR_CUDA, "pinned staging allocation of %zu bytes failed", total);
  d_imgs.resize(n);
  for (int i = 0; i < n; ++i) {
    const void* s = src[i];
    if (!host_is_pinned(src[i])) {  // pageable caller memory: stage it
      memcpy(st + offs[i], src[i], bytes[i]);
      s = st + offs[i];
    }
    PANO_CUDA(ctx, cudaMemcpyAsync(d_block + offs[i], s, bytes[i], cudaMemcpyHostToDevice, ctx->stream));
    d_imgs[i] = d_block + offs[i];
  }
  return PANO_OK;
}

// The host entry points: upload, then the device path; the uploaded block lives until the counts are
// known (a capacity retry reads it again).
static int sift_detect_host(pano_ctx* ctx, int n, const void* const* src, const int* channels, const int* w,
                            const int* h, const pano_params* p, pano_featureset** out) {
  std::vector<const void*> d_imgs;
  DevBuf<unsigned char> d_block;
  int rc = upload_images(ctx, n, src, channels, w, h, d_imgs, d_block);
  if (!rc) rc = sift_detect_dev(ctx, n, d_imgs.data(), channels, w, h, p, out);
  if (rc) return rc;
  (*out)->owned_block = std::move(d_block);
  return rc;
}

int pano_sift_detect_batch(pano_ctx* ctx, int n, const float* const* rgb, const int* w, const int* h,
                           const pano_params* p, pano_featureset** out) {
  ctx_enter(ctx);
  if (!ctx || !out || n <= 0 || !rgb || !w || !h || !p) return PANO_ERR_INVALID;
  *out = nullptr;
  return sift_detect_host(ctx, n, (const void* const*)rgb, nullptr, w, h, p, out);
}

// Checks of the 8-bit entry points: the f32 ones take any pointer, these reject what they cannot read.
// device: pix are device pointers (an RGBA source must be 4-byte aligned); host sources are staged aligned.
static int rgb8_args_ok(pano_ctx* ctx, int n, const unsigned char* const* pix, const int* w, const int* h,
                        const int* channels, const pano_params* p, bool device) {
  if (n <= 0 || !pix || !w || !h || !channels || !p) return ctx_fail(ctx, PANO_ERR_INVALID, "sift rgb8: bad argument");
  for (int i = 0; i < n; ++i) {
    if (!pix[i]) return ctx_fail(ctx, PANO_ERR_INVALID, "sift rgb8: image %d is null", i);
    if (int rc = pix8_check(ctx, "sift rgb8", i, channels[i], device ? pix[i] : nullptr)) return rc;
    if (w[i] < 2 || h[i] < 2) return ctx_fail(ctx, PANO_ERR_INVALID, "sift rgb8: image %d is %dx%d (at least 2x2)", i, w[i], h[i]);
  }
  return PANO_OK;
}

int pano_sift_detect_batch_rgb8_dev(pano_ctx* ctx, int n, const unsigned char* const* d_pix, const int* w, const int* h,
                                    const int* channels, const pano_params* p, pano_featureset** out) {
  ctx_enter(ctx);
  if (!ctx || !out) return PANO_ERR_INVALID;
  *out = nullptr;
  int rc = rgb8_args_ok(ctx, n, d_pix, w, h, channels, p, true);
  if (rc) return rc;
  return sift_detect_dev(ctx, n, (const void* const*)d_pix, channels, w, h, p, out);
}

int pano_sift_detect_batch_rgb8(pano_ctx* ctx, int n, const unsigned char* const* pix, const int* w, const int* h,
                                const int* channels, const pano_params* p, pano_featureset** out) {
  ctx_enter(ctx);
  if (!ctx || !out) return PANO_ERR_INVALID;
  *out = nullptr;
  int rc = rgb8_args_ok(ctx, n, pix, w, h, channels, p, false);
  if (rc) return rc;
  return sift_detect_host(ctx, n, (const void* const*)pix, channels, w, h, p, out);
}

int pano_sift_detect(pano_ctx* ctx, const float* rgb, int w, int h, const pano_params* p, pano_featureset** out) {
  ctx_enter(ctx);
  return pano_sift_detect_batch(ctx, 1, &rgb, &w, &h, p, out);
}

static int featureset_build(pano_ctx* ctx, int n_images, const int* n_kp, const float* const* desc,
                            const double* const* coor, pano_featureset** out, bool from_device) {
  if (!ctx || !out || n_images <= 0 || !n_kp || !desc) return PANO_ERR_INVALID;
  *out = nullptr;
  if (n_images > PANO_MAX_IMAGES)   // the matcher prepares its operands with images on gridDim.y
    return ctx_fail(ctx, PANO_ERR_INVALID, "featureset: %d images (limit %d)", n_images, PANO_MAX_IMAGES);
  std::unique_ptr<pano_featureset> fs(new pano_featureset);
  fs->ctx = ctx; fs->n_images = n_images;
  fs->base.resize(n_images); fs->h_count.resize(n_images);
  long long total = 0;
  for (int i = 0; i < n_images; ++i) {
    if (n_kp[i] < 0) return ctx_fail(ctx, PANO_ERR_INVALID, "negative count");
    fs->base[i] = total; fs->h_count[i] = n_kp[i];
    total += (n_kp[i] + 31) / 32 * 32;  // keep rows 32-aligned per image
  }
  int rc = fs->d_desc.alloc(ctx, (size_t)std::max(total, 1LL) * 128);
  if (!rc) rc = fs->d_count.alloc(ctx, n_images);
  if (!rc && coor) rc = fs->d_coor.alloc(ctx, (size_t)std::max(total, 1LL) * 2);
  if (rc) return rc;
  if (from_device) {
    // every image's rows in one launch (sources are device blocks of the exchange buffers)
    std::vector<void*> dsts; std::vector<const void*> srcs; std::vector<size_t> sizes;
    for (int i = 0; i < n_images; ++i) {
      if (!n_kp[i]) continue;
      dsts.push_back(fs->d_desc + fs->base[i] * 128); srcs.push_back(desc[i]); sizes.push_back((size_t)n_kp[i] * 128 * sizeof(float));
      if (coor && coor[i]) { dsts.push_back(fs->d_coor + fs->base[i] * 2); srcs.push_back(coor[i]); sizes.push_back((size_t)n_kp[i] * 2 * sizeof(double)); }
    }
    if ((rc = ctx_copy_blocks(ctx, (int)dsts.size(), dsts.data(), srcs.data(), sizes.data()))) return rc;
    if ((rc = ctx_put(ctx, fs->d_count, fs->h_count.data(), n_images * sizeof(int)))) return rc;
  } else {
    for (int i = 0; i < n_images; ++i) {
      if (!n_kp[i]) continue;
      PANO_CUDA(ctx, cudaMemcpyAsync(fs->d_desc + fs->base[i] * 128, desc[i], (size_t)n_kp[i] * 128 * sizeof(float),
                                     cudaMemcpyHostToDevice, ctx->stream));
      if (coor && coor[i])
        PANO_CUDA(ctx, cudaMemcpyAsync(fs->d_coor + fs->base[i] * 2, coor[i], (size_t)n_kp[i] * 2 * sizeof(double),
                                       cudaMemcpyHostToDevice, ctx->stream));
    }
    PANO_CUDA(ctx, cudaMemcpyAsync(fs->d_count, fs->h_count.data(), n_images * sizeof(int), cudaMemcpyHostToDevice, ctx->stream));
    PANO_CUDA(ctx, cudaStreamSynchronize(ctx->stream));  // sources are pageable host memory
  }
  fs->counts_on_host = true;
  *out = fs.release();
  return PANO_OK;
}

}  // extern "C"
// the same import for the communicator code (comm.cu)
int featureset_build_dev(pano_ctx* ctx, int n_images, const int* n_kp, const float* const* d_desc,
                         const double* const* d_coor, pano_featureset** out) {
  return featureset_build(ctx, n_images, n_kp, d_desc, d_coor, out, true);
}
extern "C" {

int pano_featureset_upload(pano_ctx* ctx, int n_images, const int* n_kp, const float* const* desc,
                           const double* const* coor, pano_featureset** out) {
  ctx_enter(ctx);
  return featureset_build(ctx, n_images, n_kp, desc, coor, out, false);
}

int pano_featureset_import_dev(pano_ctx* ctx, int n_images, const int* n_kp, const float* const* d_desc,
                               const double* const* d_coor, pano_featureset** out) {
  ctx_enter(ctx);
  return featureset_build(ctx, n_images, n_kp, d_desc, d_coor, out, true);
}

int pano_featureset_export_dev(pano_featureset* fs, int image, double* d_coor_xy, float* d_desc) {
  if (fs) ctx_enter(fs->ctx);
  if (!fs || image < 0 || image >= fs->n_images) return PANO_ERR_INVALID;
  int rc = featureset_sync_counts(fs);
  if (rc) return rc;
  pano_ctx* ctx = fs->ctx;
  const int n = fs->h_count[image];
  if (n == 0) return PANO_OK;
  if (d_desc) PANO_CUDA(ctx, cudaMemcpyAsync(d_desc, fs->d_desc + fs->base[image] * 128, (size_t)n * 128 * sizeof(float),
                                             cudaMemcpyDeviceToDevice, ctx->stream));
  if (d_coor_xy) {
    if (!fs->d_coor) return ctx_fail(ctx, PANO_ERR_INVALID, "featureset has no coordinates");
    PANO_CUDA(ctx, cudaMemcpyAsync(d_coor_xy, fs->d_coor + fs->base[image] * 2, (size_t)n * 2 * sizeof(double),
                                   cudaMemcpyDeviceToDevice, ctx->stream));
  }
  return PANO_OK;
}

int pano_featureset_export_all_dev(pano_featureset* fs, double* d_coor_xy, float* d_desc) {
  if (fs) ctx_enter(fs->ctx);
  if (!fs) return PANO_ERR_INVALID;
  int rc = featureset_sync_counts(fs);
  if (rc) return rc;
  pano_ctx* ctx = fs->ctx;
  if (d_coor_xy && !fs->d_coor) return ctx_fail(ctx, PANO_ERR_INVALID, "featureset has no coordinates");
  std::vector<void*> dsts; std::vector<const void*> srcs; std::vector<size_t> sizes;
  size_t off = 0;
  for (int i = 0; i < fs->n_images; ++i) {
    const size_t n = (size_t)fs->h_count[i];
    if (n && d_desc) { dsts.push_back(d_desc + off * 128); srcs.push_back(fs->d_desc + fs->base[i] * 128); sizes.push_back(n * 128 * sizeof(float)); }
    if (n && d_coor_xy) { dsts.push_back(d_coor_xy + off * 2); srcs.push_back(fs->d_coor + fs->base[i] * 2); sizes.push_back(n * 2 * sizeof(double)); }
    off += n;
  }
  return ctx_copy_blocks(ctx, (int)dsts.size(), dsts.data(), srcs.data(), sizes.data());
}

int pano_featureset_num_images(const pano_featureset* fs) {
  if (fs) ctx_enter(fs->ctx); return fs ? fs->n_images : PANO_ERR_INVALID; }

int pano_featureset_count(pano_featureset* fs, int image) {
  if (fs) ctx_enter(fs->ctx);
  if (!fs || image < 0 || image >= fs->n_images) return PANO_ERR_INVALID;
  int rc = featureset_sync_counts(fs);
  if (rc) return rc;
  return fs->h_count[image];
}

int pano_featureset_download(pano_featureset* fs, int image, double* coor_xy, float* desc) {
  if (fs) ctx_enter(fs->ctx);
  if (!fs || image < 0 || image >= fs->n_images) return PANO_ERR_INVALID;
  int rc = featureset_sync_counts(fs);
  if (rc) return rc;
  pano_ctx* ctx = fs->ctx;
  int n = fs->h_count[image];
  if (n == 0) return PANO_OK;
  if (desc) PANO_CUDA(ctx, cudaMemcpyAsync(desc, fs->d_desc + fs->base[image] * 128, (size_t)n * 128 * sizeof(float),
                                           cudaMemcpyDeviceToHost, ctx->stream));
  if (coor_xy) {
    if (!fs->d_coor) return ctx_fail(ctx, PANO_ERR_INVALID, "featureset has no coordinates");
    PANO_CUDA(ctx, cudaMemcpyAsync(coor_xy, fs->d_coor + fs->base[image] * 2, (size_t)n * 2 * sizeof(double),
                                   cudaMemcpyDeviceToHost, ctx->stream));
  }
  PANO_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return PANO_OK;
}

int pano_featureset_download_real(pano_featureset* fs, int image, double* real_xy) {
  if (fs) ctx_enter(fs->ctx);
  if (!fs || image < 0 || image >= fs->n_images || !real_xy) return PANO_ERR_INVALID;
  int rc = featureset_sync_counts(fs);
  if (rc) return rc;
  pano_ctx* ctx = fs->ctx;
  if (!fs->d_real) return ctx_fail(ctx, PANO_ERR_INVALID, "featureset was not produced by pano_sift_detect*");
  const int n = fs->h_count[image];
  if (n == 0) return PANO_OK;
  PANO_CUDA(ctx, cudaMemcpyAsync(real_xy, fs->d_real + fs->base[image] * 2, (size_t)n * 2 * sizeof(double),
                                 cudaMemcpyDeviceToHost, ctx->stream));
  PANO_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return PANO_OK;
}

void pano_featureset_free(pano_featureset* fs) {
  if (fs) ctx_enter(fs->ctx); delete fs; }

// ---------------------------------------------------------------- stage inspection

struct pano_sift_trace {
  pano_ctx* ctx;
  std::unique_ptr<SiftWork> wk;
  std::unique_ptr<pano_featureset> fs;
  DevBuf<unsigned char> d_img;
};

int pano_sift_trace_run(pano_ctx* ctx, const float* rgb, int w, int h, const pano_params* p, pano_sift_trace** out) {
  ctx_enter(ctx);
  if (!ctx || !rgb || !p || !out) return PANO_ERR_INVALID;
  *out = nullptr;
  std::vector<const void*> d_imgs;
  DevBuf<unsigned char> d_block;
  const void* src = rgb;
  int rc = upload_images(ctx, 1, &src, nullptr, &w, &h, d_imgs, d_block);
  if (rc) return rc;
  std::unique_ptr<pano_featureset> fs(new pano_featureset);
  fs->ctx = ctx;
  std::unique_ptr<SiftWork> wk;
  // the trace keeps the work buffers of ONE run, so it grows the lists itself
  for (int cap = SIFT_CAP_DEFAULT;; cap *= 2) {
    rc = sift_run_batch(ctx, 1, d_imgs.data(), nullptr, &w, &h, p, fs.get(), &wk, cap);
    if (rc) break;
    rc = featureset_sync_counts(fs.get());
    if (rc == PANO_ERR_CAPACITY && cap < SIFT_CAP_MAX) {
      wk.reset();
      fs->d_desc.reset(); fs->d_coor.reset(); fs->d_count.reset();
      fs->d_real = nullptr; fs->error = 0;
      continue;
    }
    break;
  }
  if (rc) return rc;
  *out = new pano_sift_trace{ctx, std::move(wk), std::move(fs), std::move(d_block)};
  return PANO_OK;
}

int pano_sift_trace_working_size(const pano_sift_trace* t, int* w0, int* h0) {
  if (t) ctx_enter(t->ctx);
  *w0 = t->wk->h_img[0].w0; *h0 = t->wk->h_img[0].h0;
  return PANO_OK;
}

int pano_sift_trace_octave_size(const pano_sift_trace* t, int o, int* w, int* h) {
  if (t) ctx_enter(t->ctx);
  if (o < 0 || o >= t->wk->n_oct) return PANO_ERR_INVALID;
  *w = t->wk->h_oct[o].w; *h = t->wk->h_oct[o].h;
  return PANO_OK;
}

int pano_sift_trace_plane(pano_sift_trace* t, int kind, int o, int level, float* out) {
  if (t) ctx_enter(t->ctx);
  pano_ctx* ctx = t->ctx;
  SiftWork* wk = t->wk.get();
  if (kind == 0) {
    const ImgMeta& im = wk->h_img[0];
    return pano_dev_download(ctx, out, wk->arena + im.work_off, (size_t)im.w0 * im.h0 * 3 * sizeof(float));
  }
  if (o < 0 || o >= wk->n_oct) return PANO_ERR_INVALID;
  const OctMeta& om = wk->h_oct[o];
  // planes are pitched on the device, dense for the caller
  auto download = [&](float* dst, int lvl) -> int {
    const float* src = wk->arena + om.gauss_off + (size_t)lvl * om.plane;
    PANO_CUDA(ctx, cudaMemcpy2DAsync(dst, (size_t)om.w * sizeof(float), src, (size_t)om.pitch * sizeof(float),
                                     (size_t)om.w * sizeof(float), (size_t)om.h, cudaMemcpyDeviceToHost, ctx->stream));
    PANO_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return PANO_OK;
  };
  if (kind == 1 && level >= 0 && level < wk->n_scale) return download(out, level);
  if (kind == 2 && level >= 0 && level < wk->n_scale - 1) {
    // the engine keeps no |DoG| planes: form fabsf(G(level) - G(level + 1)) as every kernel does
    const size_t np = (size_t)om.w * om.h;
    std::vector<float> next(np);
    int rc = download(out, level);
    if (rc == PANO_OK) rc = download(next.data(), level + 1);
    if (rc != PANO_OK) return rc;
    for (size_t i = 0; i < np; ++i) out[i] = fabsf(out[i] - next[i]);
    return PANO_OK;
  }
  // mag/ort are never materialised by the engine (recomputed inside the
  // orientation/descriptor kernels); not available as planes.
  return PANO_ERR_INVALID;
}

int pano_sift_trace_points(pano_sift_trace* t, int stage, int cap, pano_sspoint* out) {
  if (t) ctx_enter(t->ctx);
  pano_ctx* ctx = t->ctx;
  SiftWork* wk = t->wk.get();
  int n_raw = 0, n_desc = t->fs->h_count[0];
  if (pano_dev_download(ctx, &n_raw, wk->cand_count, sizeof(int))) return PANO_ERR_CUDA;
  n_raw = std::min(n_raw, wk->cap);
  if (stage == 0) {
    std::vector<uint32_t> keys(std::max(n_raw, 1));
    if (n_raw && pano_dev_download(ctx, keys.data(), wk->sorted_keys, n_raw * sizeof(uint32_t))) return PANO_ERR_CUDA;
    for (int i = 0; i < n_raw && i < cap; ++i) {
      memset(&out[i], 0, sizeof(pano_sspoint));
      out[i].pyr_id = keys[i] >> 29; out[i].scale_id = (keys[i] >> 26) & 7;
      out[i].y = (keys[i] >> 13) & 8191; out[i].x = keys[i] & 8191;
    }
    return n_raw;
  }
  std::vector<pano_sspoint> pts(std::max(n_raw, 1));
  std::vector<unsigned char> valid(std::max(n_raw, 1));
  if (n_raw) {
    if (pano_dev_download(ctx, pts.data(), wk->refined, n_raw * sizeof(pano_sspoint))) return PANO_ERR_CUDA;
    if (pano_dev_download(ctx, valid.data(), wk->kp_valid, n_raw)) return PANO_ERR_CUDA;
  }
  if (stage == 1) {
    int k = 0;
    for (int i = 0; i < n_raw; ++i)
      if (valid[i]) { if (k < cap) out[k] = pts[i]; ++k; }
    return k;
  }
  if (stage == 2) {
    std::vector<int> dc(std::max(n_desc, 1));
    std::vector<float> dd(std::max(n_desc, 1));
    if (n_desc) {
      if (pano_dev_download(ctx, dc.data(), wk->desc_cand, n_desc * sizeof(int))) return PANO_ERR_CUDA;
      if (pano_dev_download(ctx, dd.data(), wk->desc_dir, n_desc * sizeof(float))) return PANO_ERR_CUDA;
    }
    for (int i = 0; i < n_desc && i < cap; ++i) { out[i] = pts[dc[i]]; out[i].dir = dd[i]; }
    return n_desc;
  }
  return PANO_ERR_INVALID;
}

int pano_sift_trace_descriptors(pano_sift_trace* t, int cap, double* coor_xy, float* desc) {
  if (t) ctx_enter(t->ctx);
  int n = t->fs->h_count[0];
  if (n <= cap && n > 0) {
    int rc = pano_featureset_download(t->fs.get(), 0, coor_xy, desc);
    if (rc) return rc;
  }
  return n;
}

void pano_sift_trace_free(pano_sift_trace* t) {
  if (t) ctx_enter(t->ctx);
  delete t;
}

}  // extern "C"
