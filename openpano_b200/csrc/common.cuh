// common.cuh — context, launch/profiling helpers and the bit-exact device math
// shared by every kernel file of libpano_b200.so.
//
// Numerical contract (DESIGN.md §3): every float/double operation on the SIFT,
// match-recheck, warp and blend paths is written as the reference's compiled
// code executes it (x86-64, -ffp-contract=off): no FMA contraction (the library
// is compiled with --fmad=false), IEEE division and square root, the same
// float<->double promotions, and libm calls replaced by the exact algorithms
// glibc 2.39 runs (ARM optimized-routines expf / sinf / cosf; hypotf as
// sqrt of the double sum) so results are bit-identical, not just close.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>
#include <string>
#include <vector>
#include <algorithm>
#include <map>
#include <memory>
#include <type_traits>
#include <unordered_map>

#include "../../include/pano_b200.h"

// ------------------------------------------------------------------ owners

// Stream-ordered device memory from the CONTEXT'S OWN pool.  Contexts sharing the device's
// default pool hand each other freed blocks, and the allocator then makes the taking
// stream wait for the giving stream ("internal dependencies"): concurrent stitch lanes
// slowed down as their arenas started to cross over.
// On top of the pool sits a per-context cache of freed blocks, matched by size (best fit within
// 25 %): a stitch job asks for the same ~40 sizes every time, up to a 0.9 GB pyramid arena, and
// cudaMallocFromPoolAsync can block the host for a long time when it has to re-arrange the
// pool's mappings for such a request — with the allocator's lock held, so every other lane of
// the process stalls with it.
// Everything a context allocates is used on its one stream, so handing a block freed after its
// last enqueued use to the next request is ordered by the stream itself.  PANO_CACHE_MB bounds
// the cache (default 8192, 0 = off); pano_trim() gives the cached blocks back to the pool.
int  ctx_alloc(pano_ctx* ctx, void** p, size_t bytes);
void ctx_cache_release(pano_ctx* ctx, size_t keep_bytes);
void ctx_free(pano_ctx* ctx, void* p);
// Owner of one ctx_alloc block of T: the destructor and reset() give it back with ctx_free, so after
// everything its scope enqueued (stream order); release() hands the pointer on without freeing it.
// Reads as the raw pointer at kernel arguments and in pointer arithmetic.
template <class T>
class DevBuf {
 public:
  DevBuf() = default;
  DevBuf(pano_ctx* ctx, T* p) : ctx_(ctx), p_(p) {}   // adopts a block ctx_alloc handed out
  DevBuf(const DevBuf&) = delete;
  DevBuf& operator=(const DevBuf&) = delete;
  DevBuf(DevBuf&& o) noexcept : ctx_(o.ctx_), p_(o.release()) {}
  DevBuf& operator=(DevBuf&& o) noexcept {
    if (this != &o) { reset(); ctx_ = o.ctx_; p_ = o.release(); }
    return *this;
  }
  ~DevBuf() { reset(); }
  // `count` elements of T; a block already held is freed first
  int alloc(pano_ctx* ctx, size_t count) {
    reset();
    ctx_ = ctx;
    void* q = nullptr;
    const int rc = ctx_alloc(ctx, &q, count * sizeof(T));
    p_ = (T*)q;
    return rc;
  }
  void reset() {
    if (p_) ctx_free(ctx_, p_);
    p_ = nullptr;
  }
  T* release() { T* q = p_; p_ = nullptr; return q; }
  T* get() const { return p_; }
  operator T*() const { return p_; }

 private:
  pano_ctx* ctx_ = nullptr;
  T* p_ = nullptr;
};

// Owners of pinned host blocks, CUDA events, streams and memory pools.
struct CudaDestroy {
  void operator()(void* host) const { cudaFreeHost(host); }
  void operator()(cudaEvent_t e) const { cudaEventDestroy(e); }
  void operator()(cudaStream_t s) const { cudaStreamDestroy(s); }
  void operator()(cudaMemPool_t p) const { cudaMemPoolDestroy(p); }
};
// One page-locked host block from cudaHostAlloc (cudaFreeHost synchronises the whole device: see
// pano_ctx::small_pinned).  Move-only.
class PinnedBuf {
 public:
  // Holds at least `bytes` afterwards: a smaller block is freed and `alloc` (>= bytes) bytes are taken
  // with `flags`.  On failure the buffer is empty.
  cudaError_t grow(size_t bytes, size_t alloc, unsigned flags) {
    if (bytes <= cap()) return cudaSuccess;
    p_.reset();
    void* p = nullptr;
    const cudaError_t e = cudaHostAlloc(&p, alloc, flags);
    if (e == cudaSuccess) { p_.reset(p); cap_ = alloc; }
    return e;
  }
  void* get() const { return p_.get(); }
  size_t cap() const { return p_ ? cap_ : 0; }

 private:
  std::unique_ptr<void, CudaDestroy> p_;
  size_t cap_ = 0;   // of the block p_ holds
};
using EventPtr = std::unique_ptr<std::remove_pointer_t<cudaEvent_t>, CudaDestroy>;
using StreamPtr = std::unique_ptr<std::remove_pointer_t<cudaStream_t>, CudaDestroy>;
using PoolPtr = std::unique_ptr<std::remove_pointer_t<cudaMemPool_t>, CudaDestroy>;
static inline cudaError_t make_event(EventPtr* ev, unsigned flags) {
  cudaEvent_t e = nullptr;
  const cudaError_t err = cudaEventCreateWithFlags(&e, flags);
  ev->reset(err == cudaSuccess ? e : nullptr);
  return err;
}
static inline cudaError_t make_stream(StreamPtr* s) {
  cudaStream_t h = nullptr;
  const cudaError_t err = cudaStreamCreateWithFlags(&h, cudaStreamNonBlocking);
  s->reset(err == cudaSuccess ? h : nullptr);
  return err;
}

// ------------------------------------------------------------------ context

struct ProfEvent {
  const char* name;
  EventPtr start, stop;
};

struct SiftPlan;   // sift.cuh

struct pano_ctx {
  ~pano_ctx();
  // declared first, destroyed last: the other members may free into the pool or queue on the stream
  StreamPtr own_stream;           // the stream pano_create made; empty when it was given one (borrowed)
  cudaStream_t stream = nullptr;  // what every call of this context is queued on
  PoolPtr pool;                   // this context's own stream-ordered pool (see ctx_alloc)
  int device = 0;
  // Freed blocks kept for the next request of (about) the same size: see ctx_alloc
  struct CachedBlock { void* p; unsigned long long stamp; };
  std::multimap<size_t, CachedBlock> cache;        // size -> free block
  std::unordered_map<void*, size_t> live;           // blocks handed out -> their true size
  size_t cached_bytes = 0, cache_limit = (size_t)16 << 30;   // one 64-view multiband job parks ~8 GB; an H100 has 80
  unsigned long long cache_stamp = 0;
  std::string err;
  bool profiling = false;
  std::vector<ProfEvent> prof_pending;
  std::vector<EventPtr> event_pool;
  std::map<std::string, std::pair<int, double>> prof_acc;  // name -> (launches, ms)
  long long launches = 0;
  int last_match_exact_rows = 0;   // rows the last match call had to decide exactly (gathered pass)
  int last_match_nominated_rows = 0;   // columns on demand: rows of the larger sets nominated on request
  int last_match_full_rescans = 0; // of those, rows that needed a scan of every target
  int num_sms = 132;
  // cudaFuncSetAttribute is per device: remembered per context, never per process
  bool attr_tc = false, attr_match = false;
  int sift_cap = 0;                // per-image list capacity SIFT batches start with (grows on overflow, sticky)
  // The last SIFT batch's shape-dependent setup (sift.cu), one entry; its device bytes count against
  // cache_limit, so PANO_CACHE_MB=0 keeps none.  pano_trim, pano_destroy and ctx_alloc's
  // out-of-memory retry release it.
  std::unique_ptr<SiftPlan> sift_plan;
  void* tma_encode = nullptr;      // cuTensorMapEncodeTiled, resolved through the runtime (no -lcuda)
  // pinned host staging (grown on demand)
  PinnedBuf pinned, pinned2;
  // pinned + device-mapped ring for small host<->device moves done by SM kernels
  PinnedBuf ring;
  size_t ring_off = 0;
  // recycled pinned blocks for per-featureset count read-backs (cudaHostAlloc / cudaFreeHost
  // are slow and cudaFreeHost synchronises the whole device)
  std::vector<PinnedBuf> small_pinned;
  // completion markers: a word in pinned host memory the stream writes sequence numbers to
  PinnedBuf flag;
  unsigned flag_seq = 0;
  // planet(): per-pixel d / center and theta / 2π (planet.cu), uploaded on the first call, freed by pano_destroy
  DevBuf<double2> planet_tab;
};

// Every entry point makes its context's device current first: host threads other than the
// creating one start on device 0 (a stitch lane's thread on rank 1 would otherwise issue
// its copies against the wrong device).
static inline void ctx_enter(const pano_ctx* ctx) { if (ctx) cudaSetDevice(ctx->device); }

int  ctx_fail(pano_ctx* ctx, int code, const char* fmt, ...);
int  ctx_cuda(pano_ctx* ctx, cudaError_t e, const char* what);
void* ctx_pinned(pano_ctx* ctx, size_t bytes);   // staging buffer A (inputs)
void* ctx_pinned2(pano_ctx* ctx, size_t bytes);  // staging buffer B (results)
extern "C" bool host_is_pinned(const void* p);   // page-locked (cudaHostAlloc / pano_host_alloc) host memory
// Small host<->device moves that stay OFF the copy engines: a big image upload or
// mosaic download queued on another stream of the same device would otherwise
// delay every tiny metadata copy queued behind it on the same engine, and with it
// the kernels that depend on it.  ctx_ring reserves space in a pinned, device-
// mapped ring (valid until the ring wraps, which synchronises the stream);
// ctx_fetch / ctx_store move words with a small kernel that addresses the host
// memory directly (UVA); ctx_put = ring + memcpy + fetch; ctx_zero fills zeros.
// Host waits that SPIN on cudaEventQuery instead of sleeping in the driver: the hot
// path has two short waits per step (feature counts, match decisions) and a
// descheduled host thread on a busy machine costs milliseconds.
cudaError_t ctx_spin_event(cudaEvent_t ev);
cudaError_t ctx_spin_stream(pano_ctx* ctx);
// Short waits poll a marker word in pinned host memory instead of the driver: a host
// thread spinning in cudaEventQuery holds the context lock most of the time and starves
// another thread's kernel launches (two stitch lanes on one GPU went bimodal, 2.5 vs 5 ms).
// ctx_signal queues "write the next sequence number" on the ctx stream and returns it;
// ctx_wait_signal spins until the word has reached it (stream sync after a long timeout
// so that a device fault still surfaces).
cudaError_t ctx_signal(pano_ctx* ctx, unsigned* token);
cudaError_t ctx_wait_signal(pano_ctx* ctx, unsigned token);
void* ctx_ring(pano_ctx* ctx, size_t bytes);
// a mapped block of at least `bytes` from ctx->small_pinned (empty on failure); put gives one back to it
PinnedBuf ctx_small_pinned_get(pano_ctx* ctx, size_t bytes);
void ctx_small_pinned_put(pano_ctx* ctx, PinnedBuf&& b);
int  ctx_fetch(pano_ctx* ctx, void* d_dst, const void* h_pinned_src, size_t bytes);
int  ctx_store(pano_ctx* ctx, void* h_pinned_dst, const void* d_src, size_t bytes);
int  ctx_put(pano_ctx* ctx, void* d_dst, const void* h_src, size_t bytes);
int  ctx_zero(pano_ctx* ctx, void* d_dst, size_t bytes);
// up to CTX_MAX_SEGS moves in one launch; h_src[i] == nullptr zero-fills d_dst[i]
#define CTX_MAX_SEGS 8
int  ctx_put_many(pano_ctx* ctx, int n, void* const* d_dst, const void* const* h_src, const size_t* bytes);
int  ctx_store_many(pano_ctx* ctx, int n, void* const* h_pinned_dst, const void* const* d_src, const size_t* bytes);
int  ctx_copy_blocks(pano_ctx* ctx, int n, void* const* dst, const void* const* src, const size_t* bytes);
void ctx_prof_begin(pano_ctx* ctx, const char* name);
void ctx_prof_end(pano_ctx* ctx);

// Two-slot device ring for windows of host sources (pano_blend_stream, pano_sift_stream, pano_blend_sweep): window
// k's upload runs on the ring's own copy stream into slot k & 1 while earlier windows' kernels run on the context's
// stream; events order each slot's reuse, so at most two windows of sources are resident.  Each slot is as large as
// the largest window uploaded through it; pageable sources go through a pinned staging buffer per slot.  The copy
// stream and events are created by the first upload, so a handle given device sources only has none.
struct UploadRing {
  // the copy stream drains before the staging and slot memory go
  ~UploadRing() { if (copy) cudaStreamSynchronize(copy.get()); }
  // Uploads count host sources of bytes[k] each into the next slot and points d_src[k] at their device copies;
  // the context's stream waits for the upload.  *slot_out: the slot, to hand to release().  A failure to create
  // the copy stream or events is reported as "<what>: copy stream / events".
  int upload(pano_ctx* ctx, const char* what, int count, const void* const* srcs, const size_t* bytes,
             const void** d_src, int* slot_out);
  // The slot's last reader has been queued on the context's stream: the upload two windows on may overwrite it.
  cudaError_t release(pano_ctx* ctx, int slot);

  StreamPtr copy;
  EventPtr ev_copied[2];   // slot's upload done (copy stream)
  EventPtr ev_done[2];     // slot's last reader done (context stream)
  DevBuf<unsigned char> slot[2];
  size_t slot_cap[2] = {0, 0};
  PinnedBuf stage[2];      // pinned staging of pageable sources
  int windows = 0;         // windows uploaded so far
};

// Diagnostics (PANO_TRACE_SLOW_MS=<ms>): report every wrapped driver-facing call that blocks the host
// longer than the threshold — which call a stall sits in, not how long the GPU takes.
double pano_now_ms();
extern double g_trace_slow_ms;       // 0 = off
void pano_trace_slow(const char* what, double ms);
struct SlowCall {
  const char* what; double t0;
  explicit SlowCall(const char* w) : what(w), t0(g_trace_slow_ms > 0 ? pano_now_ms() : 0.0) {}
  ~SlowCall() { if (g_trace_slow_ms > 0) { const double d = pano_now_ms() - t0; if (d > g_trace_slow_ms) pano_trace_slow(what, d); } }
};

#define PANO_CUDA(ctx, call)                                          \
  do {                                                                \
    cudaError_t _e;                                                   \
    { SlowCall _sc(#call); _e = (call); }                             \
    if (_e != cudaSuccess) return ctx_cuda((ctx), _e, #call);         \
  } while (0)

// Launch a kernel on the ctx stream, counted and (optionally) event-timed.
#define PANO_LAUNCH(ctx, name, kernel, grid, block, smem, ...)                      \
  do {                                                                              \
    (ctx)->launches++;                                                              \
    if ((ctx)->profiling) ctx_prof_begin((ctx), (name));                            \
    { SlowCall _sc(name); kernel<<<(grid), (block), (smem), (ctx)->stream>>>(__VA_ARGS__); } \
    if ((ctx)->profiling) ctx_prof_end((ctx));                                      \
    cudaError_t _e = cudaGetLastError();                                            \
    if (_e != cudaSuccess) return ctx_cuda((ctx), _e, name);                        \
  } while (0)

// A TMA descriptor (CUtensorMap: 128 bytes, 64-byte aligned) for cp.async.bulk.tensor tile
// loads: an f32 tensor of `rank` dimensions (innermost first), strides_bytes[rank-1] for
// dimensions 1.., box = tile extent per dimension.  Encoded on the host, copied to device
// memory and handed to the kernels by pointer.
struct __align__(64) TmaDesc { unsigned long long opaque[16]; };
int ctx_tma_encode(pano_ctx* ctx, TmaDesc* out, void* base, int rank, const unsigned long long* dims,
                   const unsigned long long* strides_bytes, const unsigned* box);

// The 8-bit source formats (PANO_PIX_*, pano_b200.h): bytes per pixel, 0 for a value no 8-bit entry point
// takes.  Every 8-bit entry point, stream and staging size goes through these.
static inline int pix8_bytes(int fmt) {
  switch (fmt) {
    case PANO_PIX_GREY: return 1;
    case PANO_PIX_RGB: return 3;
    case PANO_PIX_RGBA: return 4;
    case PANO_PIX_RGB_PLANAR: return 3;
    default: return 0;
  }
}
// RGBA and planar images are read through SrcPix8; grey and interleaved RGB through SrcRgb8 (src_reader)
static inline bool pix8_layout(int fmt) { return fmt == PANO_PIX_RGBA || fmt == PANO_PIX_RGB_PLANAR; }
// Checks image i's format and, for device sources (d_pix non-null), the 4-byte alignment an RGBA tap load
// needs; fails the context with `what` in the message.
int pix8_check(pano_ctx* ctx, const char* what, int i, int fmt, const void* d_pix);

// A PANO_SRC_* kind: u8, 8-bit pixels in a PANO_PIX_* format (else h×w×3 f32); host, in host memory (else device).
struct SrcKind { int kind; bool u8, host; };
// Decodes `kind`; fails the context with `what` in the message for an unknown kind.
int src_kind(pano_ctx* ctx, const char* what, int kind, SrcKind* out);
// Bytes of a w×h source (fmt: its PANO_PIX_* format when u8)
static inline size_t src_bytes(int w, int h, bool u8, int fmt) {
  return (size_t)w * h * (u8 ? (size_t)pix8_bytes(fmt) : 3 * sizeof(float));
}
// Checks image i of a source argument: its format (a PANO_PIX_* format for 8-bit sources, 3 for f32 ones) and, for
// a device source px (null: not checked), pix8_check's alignment; fails the context with `what` in the message.
int src_check(pano_ctx* ctx, const char* what, const SrcKind& k, int i, int fmt, const void* px);

// The state every stateful handle (blend stream, SIFT stream, blend sweep, crop scan) keeps for the handle contract
// of pano_b200.h: its context, the failure that every later call returns again, and whether it has finished.
struct Sticky {
  pano_ctx* ctx = nullptr;
  int err = 0;
  bool finished = false;
  int fail(int rc) { err = rc; return rc; }
  // ctx_fail(ctx, PANO_ERR_INVALID, fmt, ...), then fail
  int misuse(const char* fmt, ...) __attribute__((format(printf, 2, 3)));
  // PANO_OK for cudaSuccess, else ctx_cuda(ctx, e, what), then fail
  int cuda(cudaError_t e, const char* what) { return e == cudaSuccess ? PANO_OK : fail(ctx_cuda(ctx, e, what)); }
  // The checks of an add of images [first, first + count) to a stream of n images that has taken `added`, in this
  // order: add after finish, the window's range, at most `cap` images in one add, the source list, a null source
  // and each source's kind and format (src_kind, src_check).  read[i] < 0 marks an image of the stream that is not
  // read (read null: all are): it needs no source and its alignment is not checked.  Messages start with `what`.
  int add_check(const char* what, int n, int added, int first, int count, int cap, const void* const* srcs,
                const int* read, int kind, int fmt, SrcKind* sk);
  // The checks of a finish after `added` of n images: a null output, a second finish, images missing; then finished.
  int finish_check(const char* what, const void* out, int added, int n);
};

// The inverse map of CylinderWarper(h_factor).warp on a w×h image (warp.cu; host arithmetic): the warped shape
// ow×oh, the constants, and the per-column tables col_x[ow] then col_cos[ow] appended to *tabs when the shape is
// not empty.  kpts (nk image-centred pairs) are rewritten in place as warp() rewrites them.  False for a
// cylinder radius <= 0.
struct CylMap { int ow, oh; double r, cy, offy, sizefactor_inv; };
bool cyl_map(int w, int h, double h_factor, const pano_params* p, double* kpts, int nk, CylMap* m,
             std::vector<double>* tabs);

static inline int ceil_div(int a, int b) { return (a + b - 1) / b; }
// gridDim.y for `count` items (at least 1 block).  CUDA refuses a grid.y above 65,535, so kernels whose
// y index is an input count (pairs, sides, segments) loop: item = blockIdx.y; item < count; item += gridDim.y.
static inline unsigned grid_y(long long count) { return (unsigned)(count < 1 ? 1 : count < 65535 ? count : 65535); }
static inline size_t align_up(size_t a, size_t b) { return (a + b - 1) / b * b; }

// Gaussian kernel exactly as GaussCache builds it (feature/gaussian.cc:17-40);
// host side, taps[0] is the tap at -center.  Returns kw.
int host_gauss_kernel(float sigma, int window_factor, float* taps, int cap);

// -------------------------------------------------------------- device math
#ifdef __CUDACC__

#define PANO_PI 3.14159265358979323846
#define PANO_PI_2 1.57079632679489661923
#define PANO_SQRT1_2 0.70710678118654752440

// lib/utils.hh:27 between(a,b,c)
#define DBETWEEN(a, b, c) (((a) >= (b)) && ((a) <= (c) - 1))

// glibc 2.39 expf (sysdeps/ieee754/flt-32/e_expf.c, ARM optimized-routines):
// x*N/ln2 = k + r, exp(x) = 2^(k/N) * p(r), N = 32, evaluated in double.
__constant__ uint64_t c_exp2f_tab[32] = {
    0x3ff0000000000000ull, 0x3fefd9b0d3158574ull, 0x3fefb5586cf9890full, 0x3fef9301d0125b51ull,
    0x3fef72b83c7d517bull, 0x3fef54873168b9aaull, 0x3fef387a6e756238ull, 0x3fef1e9df51fdee1ull,
    0x3fef06fe0a31b715ull, 0x3feef1a7373aa9cbull, 0x3feedea64c123422ull, 0x3feece086061892dull,
    0x3feebfdad5362a27ull, 0x3feeb42b569d4f82ull, 0x3feeab07dd485429ull, 0x3feea47eb03a5585ull,
    0x3feea09e667f3bcdull, 0x3fee9f75e8ec5f74ull, 0x3feea11473eb0187ull, 0x3feea589994cce13ull,
    0x3feeace5422aa0dbull, 0x3feeb737b0cdc5e5ull, 0x3feec49182a3f090ull, 0x3feed503b23e255dull,
    0x3feee89f995ad3adull, 0x3feeff76f2fb5e47ull, 0x3fef199bdd85529cull, 0x3fef3720dcef9069ull,
    0x3fef5818dcfba487ull, 0x3fef7c97337b9b5full, 0x3fefa4afa2a490daull, 0x3fefd0765b6e4540ull};

// `tab` is a 32-entry copy of c_exp2f_tab in shared memory (see load_exp2f_tab):
// lanes index it with different k, which constant memory would serialise.
__device__ __forceinline__ void load_exp2f_tab(uint64_t* s_tab, int tid) {
  if (tid < 32) s_tab[tid] = c_exp2f_tab[tid];
}

__device__ __forceinline__ float glibc_expf(float x, const uint64_t* __restrict__ tab) {
  // special ranges of the libm routine (|x| >= 88): only the underflow side can
  // occur here (arguments are -(d^2)/denom <= 0).
  if (x < -0x1.9fe368p6f) return 0.0f;
  const double InvLn2N = 0x1.71547652b82fep+0 * 32, SHIFT = 0x1.8p+52;
  const double C0 = 0x1.c6af84b912394p-5 / 32 / 32 / 32, C1 = 0x1.ebfce50fac4f3p-3 / 32 / 32,
               C2 = 0x1.62e42ff0c52d6p-1 / 32;
  double xd = (double)x;
  double z = InvLn2N * xd;
  double kd = z + SHIFT;
  uint64_t ki = (uint64_t)__double_as_longlong(kd);
  kd -= SHIFT;
  double r = z - kd;
  uint64_t t = tab[ki & 31];
  t += ki << 47;
  double s = __longlong_as_double((long long)t);
  z = C0 * r + C1;
  double r2 = r * r;
  double y = C2 * r + 1;
  y = z * r2 + y;
  y = y * s;
  return (float)y;
}

// glibc 2.39 sinf/cosf (sysdeps/ieee754/flt-32/s_sincosf.h): valid for |y| < 120.
__device__ __forceinline__ float glibc_sincos_poly(double x, double x2, bool neg_table, int n) {
  // table[1] negates the cosine coefficients only
  const double sgn = neg_table ? -1.0 : 1.0;
  if ((n & 1) == 0) {
    const double s1c = -0x1.555545995a603p-3, s2c = 0x1.1107605230bc4p-7, s3c = -0x1.994eb3774cf24p-13;
    double x3 = x * x2;
    double s1 = s2c + x2 * s3c;
    double x7 = x3 * x2;
    double s = x + x3 * s1c;
    return (float)(s + x7 * s1);
  } else {
    const double c0 = sgn * 0x1p0, c1c = sgn * -0x1.ffffffd0c621cp-2, c2c = sgn * 0x1.55553e1068f19p-5,
                 c3c = sgn * -0x1.6c087e89a359dp-10, c4c = sgn * 0x1.99343027bf8c3p-16;
    double x4 = x2 * x2;
    double c2 = c3c + x2 * c4c;
    double c1 = c1c + x2 * c2c;
    double x6 = x4 * x2;
    double c = c0 + x2 * c1;
    return (float)(c + x6 * c2);
  }
}

__device__ __forceinline__ uint32_t glibc_abstop12(float x) { return (__float_as_uint(x) >> 20) & 0x7ff; }

__device__ __forceinline__ void glibc_sincosf(float y, float* sn, float* cs) {
  const double hpi_inv = 0x1.45F306DC9C883p+23, hpi = 0x1.921FB54442D18p0;
  double x = (double)y;
  if (glibc_abstop12(y) < glibc_abstop12(0x1.921FB6p-1f)) {
    double x2 = x * x;
    if (glibc_abstop12(y) < glibc_abstop12(0x1p-12f)) { *sn = y; *cs = 1.0f; return; }
    *sn = glibc_sincos_poly(x, x2, false, 0);
    *cs = glibc_sincos_poly(x, x2, false, 1);
    return;
  }
  double r = x * hpi_inv;
  int n = ((int32_t)r + 0x800000) >> 24;
  x = x - n * hpi;
  const double sign = ((n & 3) == 1 || (n & 3) == 2) ? -1.0 : 1.0;  // {1,-1,-1,1}
  bool neg = (n & 2) != 0;
  *sn = glibc_sincos_poly(x * sign, x * x, neg, n);
  *cs = glibc_sincos_poly(x * sign, x * x, neg, n ^ 1);
}

// glibc 2.39 hypotf == (float)sqrt((double)x*x + (double)y*y) (SURVEY.md §7
// hard part 2; re-verified here on 2e7 random pairs).
__device__ __forceinline__ float glibc_hypotf(float x, float y) {
  double dx = (double)x, dy = (double)y;
  return (float)sqrt(dx * dx + dy * dy);
}

// feature/dog.cc:22-37 fast_atan
__device__ __forceinline__ float fast_atan(float y, float x) {
  float absx = fabsf(x), absy = fabsf(y);
  float m = absx > absy ? absx : absy;
  if ((double)m < 1e-6) return (float)(-PANO_PI);
  float a = (absy < absx ? absy : absx) / m;
  float s = a * a;
  double sd = (double)s, ad = (double)a;
  float r = (float)(((-0.0464964749 * sd + 0.15931422) * sd - 0.327622764) * sd * ad + ad);
  if (absy > absx) r = (float)(PANO_PI_2 - (double)r);
  if (x < 0) r = (float)(PANO_PI - (double)r);
  if (y < 0) r = -r;
  return r;
}

// feature/dog.cc:60-94 cal_mag_ort for one INTERIOR pixel (1<=x<=w-2, 1<=y<=h-2);
// border pixels have mag=0, ort=pi and are never visited by the callers.
__device__ __forceinline__ void mag_ort_at(const float* __restrict__ img, int w, int x, int y,
                                           float* mag, float* ort) {
  const float* row = img + (size_t)y * w;
  float dy = row[x + w] - row[x - w];
  float dx = row[x + 1] - row[x - 1];
  *mag = glibc_hypotf(dx, dy);
  *ort = (float)((double)fast_atan(dy, dx) + PANO_PI);
}

// Sources of the interpolate_rgb gather (tap readers, DESIGN.md §9).  at(px, w, h, fmt, lut) is the reader of one
// w×h image, its pixels px in format fmt (ignored by SrcF32) and lut the table of build_rgb8_lut (kLut readers).
// fetch gives the two horizontally adjacent pixels (fr, fc), (fr, fc + 1) and the two below them as 12 floats:
// q[0..5] row fr, q[6..11] row fr + 1.  kMayBeNo: a tap can be Color::NO; kName: the index into SRC_NAMES.
// A Mat32f, h×w×3 f32 (Color::NO = negative samples):
struct SrcF32 {
  const float* img;
  static constexpr bool kMayBeNo = true, kLut = false;
  static constexpr int kName = 0;
  static __device__ __forceinline__ SrcF32 at(const void* px, int, int, int, const float*) {
    return SrcF32{static_cast<const float*>(px)};
  }
  __device__ __forceinline__ void fetch(int w, int fr, int fc, float* q) const {
    const float* p00 = img + ((size_t)fr * w + fc) * 3;
    const float* p10 = p00 + (size_t)w * 3;
    // all twelve samples first (the four positions are in range), tests afterwards: the
    // loads overlap instead of each Color::NO test waiting on its own load
#pragma unroll
    for (int k = 0; k < 6; ++k) { q[k] = __ldg(p00 + k); q[6 + k] = __ldg(p10 + k); }
  }
};
// 8-bit pixels as read_img converts them (lib/imgio.cc:75-88, k_rgb8_to_f32): channels == 3 ->
// lut[v] = (float)((double)v / 255.0), a 256-entry table in shared memory (build_rgb8_lut);
// channels == 1 -> the grey value replicated to r, g, b WITHOUT the division.  The taps are the
// f32 values read_img would have stored, bit for bit, and never Color::NO.
struct SrcRgb8 {
  const unsigned char* pix;
  const float* lut;
  int channels;
  static constexpr bool kMayBeNo = false, kLut = true;
  static constexpr int kName = 1;
  static __device__ __forceinline__ SrcRgb8 at(const void* px, int, int, int fmt, const float* lut) {
    return SrcRgb8{static_cast<const unsigned char*>(px), lut, fmt};
  }
  __device__ __forceinline__ void fetch(int w, int fr, int fc, float* q) const {
    if (channels == 1) {
      const unsigned char* p00 = pix + (size_t)fr * w + fc;
      const float a = (float)__ldg(p00), b = (float)__ldg(p00 + 1);
      const float c = (float)__ldg(p00 + w), d = (float)__ldg(p00 + w + 1);
      q[0] = q[1] = q[2] = a; q[3] = q[4] = q[5] = b;
      q[6] = q[7] = q[8] = c; q[9] = q[10] = q[11] = d;
    } else {
      const unsigned char* p00 = pix + ((size_t)fr * w + fc) * 3;
      const unsigned char* p10 = p00 + (size_t)w * 3;
#pragma unroll
      for (int k = 0; k < 6; ++k) { q[k] = lut[__ldg(p00 + k)]; q[6 + k] = lut[__ldg(p10 + k)]; }
    }
  }
};
// 8-bit pixels in any PANO_PIX_* layout (pano_b200.h), one format per image: what a batch that holds an
// RGBA or planar image reads through (a batch of grey and interleaved RGB images keeps SrcRgb8).  RGBA is
// what lodepng::decode returns (read_png, lib/imgio.cc:43-61): every colour sample through the table, the
// fourth byte ignored, one 32-bit load per tap (the caller guarantees 4-byte alignment).  Planar is
// CImg<unsigned char>'s layout (imgio.cc:72-88): three w×h planes R, G, B, `plane` bytes apart.
struct SrcPix8 {
  const unsigned char* pix;
  const float* lut;
  int fmt;
  size_t plane;   // w * h: the planar layout's plane stride
  static constexpr bool kMayBeNo = false, kLut = true;
  static constexpr int kName = 2;
  static __device__ __forceinline__ SrcPix8 at(const void* px, int w, int h, int fmt, const float* lut) {
    return SrcPix8{static_cast<const unsigned char*>(px), lut, fmt, (size_t)w * h};
  }
  __device__ __forceinline__ void fetch(int w, int fr, int fc, float* q) const {
    if (fmt == PANO_PIX_RGBA) {
      const unsigned* p00 = reinterpret_cast<const unsigned*>(pix) + (size_t)fr * w + fc;
      const unsigned t[4] = {__ldg(p00), __ldg(p00 + 1), __ldg(p00 + w), __ldg(p00 + w + 1)};
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        q[3 * k] = lut[t[k] & 0xff]; q[3 * k + 1] = lut[(t[k] >> 8) & 0xff]; q[3 * k + 2] = lut[(t[k] >> 16) & 0xff];
      }
    } else if (fmt == PANO_PIX_RGB_PLANAR) {
      const unsigned char* p00 = pix + (size_t)fr * w + fc;
#pragma unroll
      for (int ch = 0; ch < 3; ++ch) {
        const unsigned char* p = p00 + ch * plane;
        q[ch] = lut[__ldg(p)]; q[3 + ch] = lut[__ldg(p + 1)];
        q[6 + ch] = lut[__ldg(p + w)]; q[9 + ch] = lut[__ldg(p + w + 1)];
      }
    } else {
      SrcRgb8{pix, lut, fmt}.fetch(w, fr, fc, q);
    }
  }
};
// every thread of a block of at least 256 writes one entry; the caller synchronises
__device__ __forceinline__ void build_rgb8_lut(float* lut, int tid) {
  if (tid < 256) lut[tid] = (float)((double)tid / 255.0);
}

// (int)v as x86-64 converts it (cvttss2si / cvttsd2si): toward zero, and INT_MIN for NaN and for anything
// outside [-2^31, 2^31).  A plain (int)v compiles to F2I, which saturates instead and gives 0 for NaN: where the
// reference's conversion of +inf, NaN or a value >= 2^31 yields INT_MIN, F2I would yield INT_MAX or 0.
__device__ __forceinline__ int f2i_x86(float v) {
  return (v >= -2147483648.0f && v < 2147483648.0f) ? (int)v : (int)0x80000000u;
}

// lib/imgproc.cc:135-156 interpolate; returns false for Color::NO.  Coordinates at or past 2^31, infinite or NaN
// (the inverse map of a pixel near or behind the lens horizon) floor to INT_MIN as on the host, so they fail the
// bounds test: fr + 1 never wraps and no tap is read.
template <class Src>
__device__ __forceinline__ bool interpolate_rgb(const Src& src, int w, int h, float r, float c, float* o0, float* o1,
                                                float* o2) {
  int fr = f2i_x86(floorf(r)), fc = f2i_x86(floorf(c));
  if (fr < 0 || fc < 0 || fc + 1 >= w || fr + 1 >= h) return false;
  r -= (float)fr;
  c -= (float)fc;
  float q[12];
  src.fetch(w, fr, fc, q);
  const float q00 = q[0], q01 = q[1], q02 = q[2], q03 = q[3], q04 = q[4], q05 = q[5];
  const float q10 = q[6], q11 = q[7], q12 = q[8], q13 = q[9], q14 = q[10], q15 = q[11];
  if (Src::kMayBeNo && (q00 < 0 || q10 < 0 || q13 < 0 || q03 < 0)) return false;
  float w00 = (1 - r) * (1 - c), w10 = r * (1 - c), w11 = r * c, w01 = (1 - r) * c;
  float a0 = 0.f + q00 * w00, a1 = 0.f + q01 * w00, a2 = 0.f + q02 * w00;
  a0 += q10 * w10; a1 += q11 * w10; a2 += q12 * w10;
  a0 += q13 * w11; a1 += q14 * w11; a2 += q15 * w11;
  a0 += q03 * w01; a1 += q04 * w01; a2 += q05 * w01;
  *o0 = a0; *o1 = a1; *o2 = a2;
  return true;
}
__device__ __forceinline__ bool interpolate_rgb(const float* __restrict__ img, int w, int h, float r, float c,
                                                float* o0, float* o1, float* o2) {
  return interpolate_rgb(SrcF32{img}, w, h, r, c, o0, o1, o2);
}

// One pixel (i, j) of CylinderWarper::warp's image (stitch/warp.cc:33-41) from the w×h source that src() returns
// (a tap source, made only where a tap is read): col_x / col_cos are the warp's per-column tables (warp.cu), -1
// (Color::NO) where the inverse map leaves the source.  The one statement of the warp's float and double
// operations: the stored warp (k_cyl_warp_batch) and the warp read at blend time (SrcCyl) both call it, so the two
// give the same bits.
template <class MakeSrc>
__device__ __forceinline__ void cyl_warp_px(MakeSrc src, int w, int h, const double* col_x, const double* col_cos,
                                            double r, double cy, double offy, double sizefactor_inv, int i, int j,
                                            float* o0, float* o1, float* o2) {
  double py = ((double)i - offy) * sizefactor_inv;
  double x = col_x[j];
  double y = py * r / col_cos[j] + cy;
  float v0 = -1.f, v1 = -1.f, v2 = -1.f;
  if (x >= 0 && x <= (double)(w - 1) && y >= 0 && y <= (double)(h - 1)) {
    float c0, c1, c2;
    if (interpolate_rgb(src(), w, h, (float)y, (float)x, &c0, &c1, &c2)) { v0 = c0; v1 = c1; v2 = c2; }
  }
  *o0 = v0; *o1 = v1; *o2 = v2;
}

// One image's cylinder warp as a blend reads it (pano_blend_stream_create_cyl): the unwarped source and the
// constants and device tables of its inverse map.
struct CylImg {
  const void* src;              // h×w×3 f32 or 8-bit pixels in format `channels`, as the stream's reader reads them
  int w, h;                     // the source's shape
  int channels;
  const double* col_x;          // [warped width] each
  const double* col_cos;
  double r, cy, offy, sizefactor_inv;
};

// The warped image of a CylImg as a tap source: each of the four taps is the pixel k_cyl_warp_batch would have
// stored there, computed from the source through Inner when the blend asks for it, so no warped image is ever
// held.  Unmapped pixels are Color::NO, as in the stored image.
template <class Inner>
struct SrcCyl {
  using inner_type = Inner;
  Inner src;
  const CylImg* c;
  static constexpr bool kMayBeNo = true, kLut = Inner::kLut;
  static constexpr int kName = 3 + Inner::kName;
  // px: the image's CylImg; the warped image's shape and format are not needed
  static __device__ __forceinline__ SrcCyl at(const void* px, int, int, int, const float* lut) {
    const CylImg* c = static_cast<const CylImg*>(px);
    return SrcCyl{Inner::at(c->src, c->w, c->h, c->channels, lut), c};
  }
  __device__ __forceinline__ void fetch(int, int fr, int fc, float* q) const {
    const int w = c->w, h = c->h;
    const double r = c->r, cy = c->cy, offy = c->offy, sfi = c->sizefactor_inv;
    const auto src = [this] { return this->src; };
    cyl_warp_px(src, w, h, c->col_x, c->col_cos, r, cy, offy, sfi, fr, fc, q, q + 1, q + 2);
    cyl_warp_px(src, w, h, c->col_x, c->col_cos, r, cy, offy, sfi, fr, fc + 1, q + 3, q + 4, q + 5);
    cyl_warp_px(src, w, h, c->col_x, c->col_cos, r, cy, offy, sfi, fr + 1, fc, q + 6, q + 7, q + 8);
    cyl_warp_px(src, w, h, c->col_x, c->col_cos, r, cy, offy, sfi, fr + 1, fc + 1, q + 9, q + 10, q + 11);
  }
};

// Rows [b0, b0 + rows) of an h-row f32 image (cylinder mode's mosaic band, blend_sweep.cu): `rows` holds them
// h×w×3 from row b0 on, and the reader is handed row numbers of the whole image.  The caller reads rows of the band
// only.
struct BandImg {
  const float* rows;
  int b0;
};
struct SrcBand {
  const float* img;   // row b0 of the whole image
  int b0;
  static constexpr bool kMayBeNo = true, kLut = false;
  static constexpr int kName = 6;
  // px: the BandImg
  static __device__ __forceinline__ SrcBand at(const void* px, int, int, int, const float*) {
    const BandImg* b = static_cast<const BandImg*>(px);
    return SrcBand{b->rows, b->b0};
  }
  __device__ __forceinline__ void fetch(int w, int fr, int fc, float* q) const {
    SrcF32{img + (size_t)(fr - b0) * w * 3}.fetch(w, 0, fc, q);
  }
};

// The profile name of a kernel templated on its reader: SRC_NAMES(base) lists the seven names in kName order, and
// src_name<Src> picks one.  They are literals because the profiler keeps the pointer until it drains.
#define SRC_NAMES(base) \
  {base, base "_rgb8", base "_pix8", base "_cyl", base "_cyl_rgb8", base "_cyl_pix8", base "_band"}
template <class Src> static inline const char* src_name(const char* const (&names)[7]) { return names[Src::kName]; }

// The reader of a set of formats: F32 for f32 sources (fmts null), PIX8 when one of the n formats is RGBA or
// planar, else RGB8.  with_reader(r, f) calls f(ReaderTag<Src>{}) for r's reader type Src.
enum class SrcReader { F32, RGB8, PIX8 };
template <class Src> struct ReaderTag { using type = Src; };
static inline SrcReader src_reader(const int* fmts, int n) {
  if (!fmts) return SrcReader::F32;
  return std::any_of(fmts, fmts + n, pix8_layout) ? SrcReader::PIX8 : SrcReader::RGB8;
}
template <class F>
static inline auto with_reader(SrcReader r, F&& f) {
  switch (r) {
    case SrcReader::PIX8: return f(ReaderTag<SrcPix8>{});
    case SrcReader::RGB8: return f(ReaderTag<SrcRgb8>{});
    default: return f(ReaderTag<SrcF32>{});
  }
}

#endif  // __CUDACC__
