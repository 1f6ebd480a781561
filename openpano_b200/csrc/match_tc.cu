// match_tc.cu — descriptor distance matrix on the Hopper tensor cores.
//
// The N x 128 . 128 x M contraction of the matcher (feature/matcher.cc:34-47 and
// :57-61: every query against every target, both directions) is the one GEMM of
// the hot path.  Here it runs as wgmma (f16 inputs, fp32 accumulate in registers)
// and only NOMINATES: the exact fp32 rule of the reference is then decided
// by match.cu from certified bounds, with an exact re-scan of the few ambiguous
// rows, so the match pairs stay bit-identical.
//
// Operands.  k_tc_prep converts every descriptor x (f32[128]) into two fp16 rows
// of K = 144 (128 + one extra 16-wide k-step):
//     query  form: [ s*x        | 1, 1, n_hi, n_lo, 1, 0... ]
//     target form: [ -2*s*x     | n_hi, n_lo, 1, 1, 1, 0... ]     n = s^2*|x|^2
// so that  q . t ~ s^2 * |xq - xt|^2 + 1.  s is a power of two making n <= 1024 (s = 1/16 for RootSIFT,
// |x| = 512).  The score is NOT always positive: with f = fp16(s*x), q . t = s^2 |fq - ft|^2 + 1
// + (nq - |fq|^2) + (nt - |ft|^2), and each bracket reaches -n/1024, so a row against a near-duplicate of
// itself scores down to 1 - n/512 (-1 at n = 1024; ~-0.98 for rows whose components all sit just above
// fp16 midpoints).  Negative scores order backwards as signed-int keys, so among two such targets the
// top-2 may nominate the worse as best, with m2 < m1.  The decision stays exact because every
// approximate distance lies within tc_eps of the exact one, and m + tc_eps > 0 for every reachable m:
// refine_row then finds the argmin uncertain, keeps lower bounds of 0 and positive upper bounds, and the
// row is re-scanned exactly.  Until then its bounds also serve as a column's bounds in k_match_decide,
// where sec_hi = m2 + eps can lie below min_{kk != k} d(j, kk) when k is the column behind m2.  That
// bound can only reject row k (its lower bound c_lo is 0), and every row k it rejects is one the
// reference rejects too; the filter threshold m2 + 2.5 eps still covers every column that can be the
// exact best or second best (|m1 - m2| stays below eps / 2).  tests/test_match_bound.py checks these
// facts on the operands of k_tc_prep; tests/test_gpu_match_warp_blend.py runs such rows on the device.
// Rows are stored PRE-BLOCKED in the canonical K-major no-swizzle layout of wgmma shared-memory
// operands (8x16-byte core matrices, SBO = 128 B): query rows in 128-row blocks (LBO = 2 KiB),
// target rows in 256-row tiles (LBO = 4 KiB), so one contiguous cp.async.bulk brings a block / tile
// into shared memory ready for the MMA.
//
// Kernel k_tc_pass, persistent, one CTA per SM walking tasks = (query block of 128 rows) x (a range
// of target tiles):
//   warpgroup 0    producer : one thread issues cp.async.bulk of target tiles (256 rows, 72 KiB) into
//                             a 2-stage ring and of query blocks into two buffers (mbarrier transactions)
//   warpgroups 1-2 consumers: warpgroup c owns query rows [64 c, 64 c + 64) of the block.  Per tile it
//                             issues 2 x 9 wgmma m64n128k16 (one group per 128-column half, both read
//                             shared memory directly), and reduces the first half while the second is
//                             still in flight; while one warpgroup reduces, the other one's MMAs run.
//                             A thread holds two rows x 32 columns of each half (the wgmma accumulator
//                             layout) and keeps a running (min, argmin, second-min) per row with the
//                             column packed into the low mantissa bits (one LOP3 and 1.5 VIMNMX per
//                             element); on long target sets a half whose minimum is not below the
//                             thread's running second best is skipped.  The four threads sharing a row
//                             merge their top-2 through shuffles once per task.
#include "sift.cuh"
#include "match_tc.cuh"
#include <cuda_fp16.h>
#include <float.h>
#include <algorithm>

#define TC_KC 18                       // 16-byte k-chunks per row: 144 fp16
#define TC_BLOCK_BYTES (TC_KC * 2048)  // 128 rows x 144 fp16 = 36864 B
#define TC_LBO 2048u                   // byte stride between k-chunks (128-row query blocks)
#define TC_TLBO 4096u                  // the same for the 256-row target tiles
#define TC_SBO 128u                    // byte stride between 8-row groups
#define TC_TILE_BLOCKS 2               // target tile = 2 blocks = 256 rows
#define TC_STAGES 2
#define TC_THREADS 384              // warpgroup 0: producer; warpgroups 1, 2: consumers
#define TC_CONSUMER_WARPS 8

// ------------------------------------------------------------------ prep

__global__ void k_tc_maxnorm(const float* __restrict__ desc, const TcImage* __restrict__ imgs, int n_img,
                             float* __restrict__ norms, unsigned* __restrict__ maxnorm_bits) {
  const int img = blockIdx.y;
  const TcImage im = imgs[img];
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  float n = 0.f;
  if (r < im.n) {
    const float4* p = (const float4*)(desc + (size_t)(im.row0 + r) * 128);
    float acc = 0.f;
#pragma unroll 8
    for (int k = 0; k < 32; ++k) { float4 v = __ldg(p + k); acc += v.x * v.x; acc += v.y * v.y; acc += v.z * v.z; acc += v.w * v.w; }
    n = acc;
    norms[im.row0 + r] = n;
  }
  // block max -> global max (floats >= 0 order like unsigned ints)
  for (int off = 16; off; off >>= 1) n = fmaxf(n, __shfl_xor_sync(0xffffffffu, n, off));
  if ((threadIdx.x & 31) == 0 && n > 0.f) atomicMax(maxnorm_bits, __float_as_uint(n));
}

__device__ __forceinline__ float tc_scale_from_maxnorm(float maxn2) {
  // s = 2^-e with s^2 * maxn2 <= 1024
  if (!(maxn2 > 0.f)) return 1.f;
  int e = (int)ceilf(0.5f * log2f(maxn2 / 1024.f));
  return exp2f((float)-e);
}

// one thread per (row, form): writes 18 16-byte chunks into the blocked layout
__global__ void k_tc_prep(const float* __restrict__ desc, const float* __restrict__ norms,
                          const unsigned* __restrict__ maxnorm_bits, const TcImage* __restrict__ imgs,
                          unsigned char* __restrict__ qbuf, unsigned char* __restrict__ tbuf) {
  const TcImage im = imgs[blockIdx.y];
  const int r = blockIdx.x * blockDim.x + threadIdx.x;   // padded row index
  if (r >= im.n_pad) return;
  const float s = tc_scale_from_maxnorm(__uint_as_float(*maxnorm_bits));
  const size_t blk = (size_t)(im.blk0 + r / 128);
  const int rr = r % 128;
  unsigned char* qd = qbuf + blk * TC_BLOCK_BYTES + (rr / 8) * TC_SBO + (rr % 8) * 16;
  // targets are laid out in 256-ROW tiles (one N = 256 MMA reads a whole tile: 32 row groups at SBO
  // per k-chunk, k-chunks TC_TLBO apart); n_pad is a multiple of 256, so tile t of an image starts
  // at block blk0 + 2 t either way
  const int tr = r % 256;
  unsigned char* td = tbuf + (size_t)(im.blk0 + (r / 256) * 2) * TC_BLOCK_BYTES + (tr / 8) * TC_SBO + (tr % 8) * 16;
  const bool real = r < im.n;
  const float4* p = (const float4*)(desc + (size_t)(im.row0 + (real ? r : 0)) * 128);
#pragma unroll 4
  for (int kc = 0; kc < 16; ++kc) {
    float4 a = real ? __ldg(p + 2 * kc) : make_float4(0.f, 0.f, 0.f, 0.f);
    float4 b = real ? __ldg(p + 2 * kc + 1) : make_float4(0.f, 0.f, 0.f, 0.f);
    __half2 q0 = __floats2half2_rn(a.x * s, a.y * s), q1 = __floats2half2_rn(a.z * s, a.w * s);
    __half2 q2 = __floats2half2_rn(b.x * s, b.y * s), q3 = __floats2half2_rn(b.z * s, b.w * s);
    const float m = -2.f * s;
    __half2 t0 = __floats2half2_rn(a.x * m, a.y * m), t1 = __floats2half2_rn(a.z * m, a.w * m);
    __half2 t2 = __floats2half2_rn(b.x * m, b.y * m), t3 = __floats2half2_rn(b.z * m, b.w * m);
    uint4 qv, tv;
    qv.x = *(unsigned*)&q0; qv.y = *(unsigned*)&q1; qv.z = *(unsigned*)&q2; qv.w = *(unsigned*)&q3;
    tv.x = *(unsigned*)&t0; tv.y = *(unsigned*)&t1; tv.z = *(unsigned*)&t2; tv.w = *(unsigned*)&t3;
    *(uint4*)(qd + (size_t)kc * TC_LBO) = qv;
    *(uint4*)(td + (size_t)kc * TC_TLBO) = tv;
  }
  // extra k-step: chunks 16 and 17
  float n = real ? norms[im.row0 + r] * s * s : 0.f;
  __half nh = __float2half_rn(n);
  __half nl = __float2half_rn(n - __half2float(nh));
  const __half one = __float2half_rn(1.f), zero = __float2half_rn(0.f);
  __half qx[8] = {one, one, nh, nl, one, zero, zero, zero};
  __half tx[8] = {nh, nl, one, one, one, zero, zero, zero};
  if (!real) {  // padded target rows must never win: q.t = 30000
    tx[0] = __float2half_rn(30000.f); tx[1] = zero; tx[2] = zero; tx[3] = zero; tx[4] = zero;
    qx[2] = zero; qx[3] = zero;
  }
  *(uint4*)(qd + (size_t)16 * TC_LBO) = *(uint4*)qx;
  *(uint4*)(td + (size_t)16 * TC_TLBO) = *(uint4*)tx;
  *(uint4*)(qd + (size_t)17 * TC_LBO) = make_uint4(0, 0, 0, 0);
  *(uint4*)(td + (size_t)17 * TC_TLBO) = make_uint4(0, 0, 0, 0);
}

// ------------------------------------------------------------------ PTX helpers

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
// Bounded wait: a protocol bug traps instead of hanging the GPU.
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  uint32_t done = 0;
  for (uint32_t spin = 0; spin < (1u << 28); ++spin) {
    asm volatile(
        "{\n\t.reg .pred P1;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 P1, [%1], %2;\n\t"
        "selp.b32 %0, 1, 0, P1;\n\t}"
        : "=r"(done)
        : "r"(bar), "r"(parity)
        : "memory");
    if (done) return;
  }
  __trap();
}
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t saddr, uint32_t lbo) {
  // wgmma matrix descriptor (K-major, no swizzle): start>>4 [0,14), LBO>>4 [16,30), SBO>>4 [32,46)
  return (uint64_t)((saddr & 0x3FFFFu) >> 4) | ((uint64_t)(lbo >> 4) << 16) | ((uint64_t)(TC_SBO >> 4) << 32);
}
// D[64 x 128] (+)= A[64 x 16] . B[128 x 16]^T, both operands K-major in shared memory
__device__ __forceinline__ void wgmma_m64n128k16(float (&d)[64], uint64_t adesc, uint64_t bdesc, int accum) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "%64, %65, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(adesc), "l"(bdesc), "r"(accum));
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator reads / writes across the asynchronous MMA
__device__ __forceinline__ void acc_fence(float (&d)[64]) {
#pragma unroll
  for (int i = 0; i < 64; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// ------------------------------------------------------------------ the GEMM + top-2 kernel

struct __align__(8) TcBarriers {
  uint64_t full[TC_STAGES], empty[TC_STAGES], a_full[2], a_empty[2];
};

// One half (128 target columns) of a tile in a consumer thread's accumulators: element 4i + e holds
// row r0 (e < 2) or r0 + 8 (e >= 2), column 128 h + 8 i + 2 quad + (e & 1).  The key packs the column
// WITHOUT the 2 quad term (the same for every element of the thread) so that it stays an immediate;
// the term is added back when the key's column is read out.
template <bool FILTER, int H>
__device__ __forceinline__ void tc_reduce_half(const float (&d)[64], uint32_t keymask, bool prefilter, const int* g2,
                                               int* k1, int* k2, const int* thr, int col_base, int t_n, const int* grow,
                                               int* __restrict__ cand_cnt, int* __restrict__ cand) {
  if (FILTER) {
    // branch-free hit masks first: a conditional body inside the unrolled compare blows the loop
    // up past the instruction cache
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      unsigned hit = 0;
#pragma unroll
      for (int j = 0; j < 32; ++j)
        hit |= ((int)(__float_as_uint(d[4 * (j >> 1) + 2 * r + (j & 1)]) & 0xffffff00u) <= thr[r]) ? (1u << j) : 0u;
      while (hit) {
        const int j = __ffs(hit) - 1;
        hit &= hit - 1;
        const int col = col_base + H * 128 + 8 * (j >> 1) + (j & 1);
        if (col < t_n) {
          const int slot = atomicAdd(&cand_cnt[grow[r]], 1);
          if (slot < TC_CAND_CAP) cand[(size_t)grow[r] * TC_CAND_CAP + slot] = col;
        }
      }
    }
  } else {
    if (prefilter) {
      // A half none of whose scores is below the thread's running second best cannot change its
      // top-2 (masking is monotone, ties keep the earlier column); with c columns seen, a row
      // improves in a half with probability ~2/c, so on long target sets most halves are skipped.
      int m0 = (int)__float_as_uint(d[0]), m1 = (int)__float_as_uint(d[2]);
#pragma unroll
      for (int i = 0; i < 16; ++i) {
        m0 = min(m0, min((int)__float_as_uint(d[4 * i]), (int)__float_as_uint(d[4 * i + 1])));
        m1 = min(m1, min((int)__float_as_uint(d[4 * i + 2]), (int)__float_as_uint(d[4 * i + 3])));
      }
      if (!__any_sync(0xffffffffu, m0 < g2[0] || m1 < g2[1])) return;
    }
#pragma unroll
    for (int i = 0; i < 16; ++i)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        // (v & mask) | column in ONE LOP3: the mask has to sit in a register, because the
        // instruction takes a single immediate
        uint32_t ukey;
        asm("lop3.b32 %0, %1, %2, %3, 0xEA;" : "=r"(ukey) : "r"(__float_as_uint(d[4 * i + e])), "r"(keymask), "r"((uint32_t)(H * 128 + 8 * i + (e & 1))));
        const int key = (int)ukey, r = e >> 1;
        k2[r] = min(k2[r], max(k1[r], key));
        k1[r] = min(k1[r], key);
      }
  }
}

// FILTER = false: running top-2 per query row (the nomination pass).
// FILTER = true : second pass over GATHERED rows only; every column whose score is
//                 within the row's threshold key is appended to that row's candidate
//                 slots (the exact kernel then decides among a handful of columns).
//
// PERSISTENT: a CTA walks tasks blockIdx.x, blockIdx.x + gridDim.x, ...; the producer and the two
// consumer warpgroups run the same task sequence on their own, coupled only through mbarriers whose
// phases follow two running counters (target tiles and tasks).  Nothing is re-initialised between
// tasks, so the producer is already fetching the next task's query block (two A buffers) and target
// tiles while the consumers finish the current one: an image pair of ~2 k descriptors is only ~10
// tiles per task.
template <bool FILTER>
__global__ void __launch_bounds__(TC_THREADS, 1)
k_tc_pass(const unsigned char* __restrict__ qbuf, const unsigned char* __restrict__ tbuf,
          const TcTask* __restrict__ tasks, const int* __restrict__ n_tasks_dev, int n_tasks_host,
          const unsigned* __restrict__ maxnorm_bits, TcTop2* __restrict__ res,
          const int* __restrict__ g_thr, int* __restrict__ cand_cnt, int* __restrict__ cand) {
  extern __shared__ __align__(1024) unsigned char tc_smem[];
  const int task_end = n_tasks_dev ? *n_tasks_dev : n_tasks_host;
  if ((int)blockIdx.x >= task_end) return;   // uniform per CTA, before any barrier use
  unsigned char* sA = tc_smem;                                        // 2 query blocks
  unsigned char* sB = tc_smem + 2 * TC_BLOCK_BYTES;                   // TC_STAGES x 2 blocks
  TcBarriers* bars = (TcBarriers*)(sB + (size_t)TC_STAGES * TC_TILE_BLOCKS * TC_BLOCK_BYTES);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    // the consumers release a buffer with one arrival per warp, after that warp's wgmma.wait_group
    for (int s = 0; s < TC_STAGES; ++s) { mbar_init(smem_u32(&bars->full[s]), 1); mbar_init(smem_u32(&bars->empty[s]), TC_CONSUMER_WARPS); }
    for (int s = 0; s < 2; ++s) { mbar_init(smem_u32(&bars->a_full[s]), 1); mbar_init(smem_u32(&bars->a_empty[s]), TC_CONSUMER_WARPS); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp == 0) {
    // ===== producer
    if (lane == 0) {
      uint32_t gt = 0;                       // target tiles issued so far (all tasks)
      uint32_t ti = 0;                       // tasks started so far
      for (int task = blockIdx.x; task < task_end; task += gridDim.x, ++ti) {
        const TcTask tk = tasks[task];
        const int ntile = tk.t_blocks / TC_TILE_BLOCKS;
        const uint32_t as = ti & 1u;
        mbar_wait(smem_u32(&bars->a_empty[as]), ((ti >> 1) & 1u) ^ 1u);
        mbar_expect_tx(smem_u32(&bars->a_full[as]), TC_BLOCK_BYTES);
        bulk_g2s(smem_u32(sA + (size_t)as * TC_BLOCK_BYTES), qbuf + (size_t)tk.q_blk * TC_BLOCK_BYTES, TC_BLOCK_BYTES,
                 smem_u32(&bars->a_full[as]));
        for (int t = 0; t < ntile; ++t, ++gt) {
          const uint32_t s = gt % TC_STAGES, ph = (gt / TC_STAGES) & 1u;
          mbar_wait(smem_u32(&bars->empty[s]), ph ^ 1u);
          const uint32_t bytes = TC_TILE_BLOCKS * TC_BLOCK_BYTES;
          mbar_expect_tx(smem_u32(&bars->full[s]), bytes);
          bulk_g2s(smem_u32(sB + (size_t)s * bytes), tbuf + (size_t)(tk.t_blk0 + t * TC_TILE_BLOCKS) * TC_BLOCK_BYTES, bytes,
                   smem_u32(&bars->full[s]));
        }
      }
    }
  } else if (warp >= 4) {
    // ===== consumers: warpgroup wg = query rows [64 wg, 64 wg + 64); thread <-> rows r0, r0 + 8
    const int wg = (warp - 4) >> 2, quad = lane & 3;
    const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);
    const int rows[2] = {r0, r0 + 8};
    uint32_t keymask;
    asm volatile("mov.b32 %0, 0xffffff00;" : "=r"(keymask));
    float acc0[64], acc1[64];
    uint32_t gt = 0, ti = 0;
    for (int task = blockIdx.x; task < task_end; task += gridDim.x, ++ti) {
      const TcTask tk = tasks[task];
      const int ntile = tk.t_blocks / TC_TILE_BLOCKS;
      int g1[2] = {0x7f7fff00, 0x7f7fff00}, g2[2] = {0x7f7fff00, 0x7f7fff00};   // running best / second (value bits, low 8 cleared)
      int gi[2] = {0x7fffffff, 0x7fffffff};
      const int col0 = (FILTER || n_tasks_dev) ? 0 : tk.t_pad;   // first pass: first column of this task's range
      int grow[2], thr[2];                      // FILTER: index of each row among the gathered rows, its threshold
#pragma unroll
      for (int r = 0; r < 2; ++r) { grow[r] = tk.q_row0 + rows[r]; thr[r] = FILTER ? g_thr[grow[r]] : 0; }
      // long target sets only: on short ones nearly every half still improves some row of the warp
      const bool prefilter = !FILTER && tk.t_blocks >= 128;
      const uint32_t asl = ti & 1u;
      mbar_wait(smem_u32(&bars->a_full[asl]), (ti >> 1) & 1u);
      const uint32_t a0 = smem_u32(sA + (size_t)asl * TC_BLOCK_BYTES) + (uint32_t)(wg * 8) * TC_SBO;
      for (int t = 0; t < ntile; ++t, ++gt) {
        const uint32_t s = gt % TC_STAGES;
        mbar_wait(smem_u32(&bars->full[s]), (gt / TC_STAGES) & 1u);
        const uint32_t b0 = smem_u32(sB + (size_t)s * TC_TILE_BLOCKS * TC_BLOCK_BYTES);
        acc_fence(acc0); acc_fence(acc1);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < TC_KC / 2; ++k)
          wgmma_m64n128k16(acc0, make_smem_desc(a0 + k * 2 * TC_LBO, TC_LBO), make_smem_desc(b0 + k * 2 * TC_TLBO, TC_TLBO), k);
        wgmma_commit();
#pragma unroll
        for (int k = 0; k < TC_KC / 2; ++k)   // target rows 128-255 of the tile: row groups 16-31
          wgmma_m64n128k16(acc1, make_smem_desc(a0 + k * 2 * TC_LBO, TC_LBO),
                           make_smem_desc(b0 + 16 * TC_SBO + k * 2 * TC_TLBO, TC_TLBO), k);
        wgmma_commit();
        int k1[2] = {0x7fffffff, 0x7fffffff}, k2[2] = {0x7fffffff, 0x7fffffff};
        const int col_base = t * 256 + 2 * quad;
        wgmma_wait<1>();
        acc_fence(acc0);
        tc_reduce_half<FILTER, 0>(acc0, keymask, prefilter, g2, k1, k2, thr, col_base, tk.t_n, grow, cand_cnt, cand);
        wgmma_wait<0>();
        acc_fence(acc1);
        __syncwarp();
        if (lane == 0) mbar_arrive(smem_u32(&bars->empty[s]));   // this warp's MMAs have read the stage
        tc_reduce_half<FILTER, 1>(acc1, keymask, prefilter, g2, k1, k2, thr, col_base, tk.t_n, grow, cand_cnt, cand);
        if (!FILTER) {
          // merge the tile's top-2 into the running top-2 (an earlier tile wins a tie: lower column)
#pragma unroll
          for (int r = 0; r < 2; ++r) {
            const int v1 = k1[r] & (int)0xffffff00, v2 = k2[r] & (int)0xffffff00;
            if (v1 < g1[r]) { g2[r] = min(g1[r], v2); g1[r] = v1; gi[r] = col0 + col_base + (k1[r] & 0xff); }
            else g2[r] = min(g2[r], v1);
          }
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(smem_u32(&bars->a_empty[asl]));   // every MMA of this warp that reads the query block is done
#pragma unroll
      for (int r = 0; r < 2 && !FILTER; ++r) {
        // the four threads of a row hold interleaved columns: equal scores keep the lower column
#pragma unroll
        for (int off = 1; off < 4; off <<= 1) {
          const int o1 = __shfl_xor_sync(0xffffffffu, g1[r], off), o2 = __shfl_xor_sync(0xffffffffu, g2[r], off);
          const int oi = __shfl_xor_sync(0xffffffffu, gi[r], off);
          if (o1 < g1[r] || (o1 == g1[r] && oi < gi[r])) { g2[r] = min(g1[r], o2); g1[r] = o1; gi[r] = oi; }
          else g2[r] = min(g2[r], o1);
        }
        // device-planned tasks (n_tasks_dev) are GATHERED blocks: q_row0 is the block's first gathered
        // row, q_n its real rows, and the nomination goes to the gathered row's slot
        const int qrow = tk.q_row0 + rows[r];
        if (quad == 0 && (n_tasks_dev ? rows[r] < tk.q_n : qrow < tk.q_n)) {
          const float s = tc_scale_from_maxnorm(__uint_as_float(*maxnorm_bits));
          const float inv = 1.f / (s * s);
          TcTop2 o;
          o.m1 = (__int_as_float(g1[r]) - 1.f) * inv;
          o.m2 = g2[r] == 0x7f7fff00 ? FLT_MAX : (__int_as_float(g2[r]) - 1.f) * inv;
          o.idx = gi[r];
          o.pad = 0;
          res[(n_tasks_dev ? 0 : tk.res_off) + qrow] = o;
        }
      }
    }
  }
}

// ------------------------------------------------------------------ host side

size_t tc_block_bytes() { return TC_BLOCK_BYTES; }

size_t tc_smem_bytes() {
  return (size_t)TC_BLOCK_BYTES * (2 + TC_STAGES * TC_TILE_BLOCKS) + sizeof(TcBarriers) + 1024;
}

int tc_prepare(pano_ctx* ctx, const float* d_desc, const std::vector<TcImage>& imgs, TcOperands* ops) {
  const int n = (int)imgs.size();
  long long rows = 0, blocks = 0;
  int max_pad = 0;
  for (auto& im : imgs) { rows = std::max<long long>(rows, im.row0 + im.n); blocks = std::max<long long>(blocks, im.blk0 + im.n_pad / 128); max_pad = std::max(max_pad, im.n_pad); }
  int rc = 0;
  if ((rc = ops->d_imgs.alloc(ctx, n)) || (rc = ops->d_norms.alloc(ctx, std::max<long long>(rows, 1))) ||
      (rc = ops->d_maxnorm.alloc(ctx, 1)) ||
      (rc = ops->qbuf.alloc(ctx, (size_t)std::max<long long>(blocks, 1) * TC_BLOCK_BYTES)) ||
      (rc = ops->tbuf.alloc(ctx, (size_t)std::max<long long>(blocks, 1) * TC_BLOCK_BYTES)))
    return rc;
  if ((rc = ctx_put(ctx, ops->d_imgs, imgs.data(), n * sizeof(TcImage)))) return rc;
  if ((rc = ctx_zero(ctx, ops->d_maxnorm, sizeof(unsigned)))) return rc;
  if (max_pad == 0) return PANO_OK;
  dim3 g1(ceil_div(max_pad, 128), n);
  PANO_LAUNCH(ctx, "k_tc_maxnorm", k_tc_maxnorm, g1, 128, 0, d_desc, ops->d_imgs, n, ops->d_norms, ops->d_maxnorm);
  PANO_LAUNCH(ctx, "k_tc_prep", k_tc_prep, g1, 128, 0, d_desc, ops->d_norms, ops->d_maxnorm, ops->d_imgs, ops->qbuf, ops->tbuf);
  return PANO_OK;
}

// function attributes are per DEVICE: one process may hold contexts on several GPUs
static int tc_set_attrs(pano_ctx* ctx) {
  if (ctx->attr_tc) return PANO_OK;
  const size_t smem = tc_smem_bytes();
  PANO_CUDA(ctx, cudaFuncSetAttribute(k_tc_pass<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  PANO_CUDA(ctx, cudaFuncSetAttribute(k_tc_pass<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  ctx->attr_tc = true;
  return PANO_OK;
}

int tc_run_top2(pano_ctx* ctx, const TcOperands* ops, const TcTask* d_tasks, int n_tasks, TcTop2* d_res) {
  if (n_tasks == 0) return PANO_OK;
  const size_t smem = tc_smem_bytes();
  if (int rc = tc_set_attrs(ctx)) return rc;
  PANO_LAUNCH(ctx, "k_tc_top2", k_tc_pass<false>, std::min(n_tasks, ctx->num_sms), TC_THREADS, smem, ops->qbuf, ops->tbuf, d_tasks,
              (const int*)nullptr, n_tasks, ops->d_maxnorm, d_res, (const int*)nullptr, (int*)nullptr, (int*)nullptr);
  return PANO_OK;
}

// ------------------------------------------------------------------ gathered second pass

// Copies the query-form fp16 rows of the listed rows into gather blocks and sets
// each gathered row's threshold key / bookkeeping (approx == nullptr: a nomination pass over
// rows that have no first-pass result yet — no thresholds).  One CTA per gather block.
__global__ void __launch_bounds__(128)
k_tc_gather_rows(const unsigned char* __restrict__ qbuf, unsigned char* __restrict__ gq,
                 const TcTask* __restrict__ tasks, const int* __restrict__ n_tasks_dev,
                 const TcGatherSide* __restrict__ gsides, const int* __restrict__ list_rows,
                 const TcTop2* __restrict__ approx, const float* __restrict__ norms,
                 const unsigned* __restrict__ maxnorm_bits, int2* __restrict__ g_meta, int* __restrict__ g_thr,
                 int* __restrict__ cand_cnt) {
  if ((int)blockIdx.x >= *n_tasks_dev) return;
  const TcTask tk = tasks[blockIdx.x];
  const int side = (int)tk.res_off;                 // filter tasks carry the side index here
  const TcGatherSide gs = gsides[side];
  const int r = threadIdx.x, g = tk.q_row0 + r;
  unsigned char* dst = gq + (size_t)tk.q_blk * TC_BLOCK_BYTES + (r / 8) * TC_SBO + (r % 8) * 16;
  if (r < tk.q_n) {
    const int row = list_rows[gs.list_off + tk.t_pad + r];      // t_pad = first list slot of this block
    const unsigned char* src = qbuf + (size_t)(gs.q_blk0 + row / 128) * TC_BLOCK_BYTES + ((row % 128) / 8) * TC_SBO + (row % 8) * 16;
#pragma unroll
    for (int kc = 0; kc < TC_KC; ++kc) *(uint4*)(dst + (size_t)kc * TC_LBO) = *(const uint4*)(src + (size_t)kc * TC_LBO);
    if (approx) {
      const float nmax = __uint_as_float(*maxnorm_bits);
      const float s = tc_scale_from_maxnorm(nmax);
      const float nq = norms[gs.q_base + row];
      const float eps = 0.00215f * sqrtf(nq * nmax) + 0.0005f * nmax + 1.0f;    // == tc_eps in match.cu
      const TcTop2 ap = approx[gs.res_off + row];
      // every column whose exact distance can be the best or the second best scores <= m2~ + 2 eps
      float thr_v = ap.m2 == FLT_MAX ? FLT_MAX : (ap.m2 + 2.5f * eps) * (s * s) + 1.f;
      g_thr[g] = (int)(__float_as_uint(thr_v) | 0xffu);
      cand_cnt[g] = 0;
    }
    g_meta[g] = make_int2(side, row);
  } else {
#pragma unroll
    for (int kc = 0; kc < TC_KC; ++kc) *(uint4*)(dst + (size_t)kc * TC_LBO) = make_uint4(0, 0, 0, 0);
    if (approx) { g_thr[g] = -1; cand_cnt[g] = 0; }
    g_meta[g] = make_int2(-1, -1);
  }
}

int tc_run_filter(pano_ctx* ctx, const TcOperands* ops, const TcFilter* f, int max_blocks) {
  if (max_blocks <= 0) return PANO_OK;
  const size_t smem = tc_smem_bytes();
  if (int rc = tc_set_attrs(ctx)) return rc;
  PANO_LAUNCH(ctx, "k_tc_gather_rows", k_tc_gather_rows, max_blocks, 128, 0, ops->qbuf, f->gq, f->tasks, f->n_tasks,
              f->gsides, f->list_rows, f->approx, ops->d_norms, ops->d_maxnorm, f->g_meta, f->g_thr, f->cand_cnt);
  PANO_LAUNCH(ctx, "k_tc_filter", k_tc_pass<true>, std::min(max_blocks, ctx->num_sms), TC_THREADS, smem, f->gq, ops->tbuf, f->tasks, f->n_tasks,
              0, ops->d_maxnorm, (TcTop2*)nullptr, f->g_thr, f->cand_cnt, f->cand);
  return PANO_OK;
}

// Nomination (running top-2) over gathered rows: the columns-on-demand pass of match.cu.
// d_res[g] receives gathered row g's result.
int tc_run_nominate(pano_ctx* ctx, const TcOperands* ops, const TcFilter* f, int max_blocks, TcTop2* d_res) {
  if (max_blocks <= 0) return PANO_OK;
  const size_t smem = tc_smem_bytes();
  if (int rc = tc_set_attrs(ctx)) return rc;
  PANO_LAUNCH(ctx, "k_tc_gather_rows", k_tc_gather_rows, max_blocks, 128, 0, ops->qbuf, f->gq, f->tasks, f->n_tasks,
              f->gsides, f->list_rows, (const TcTop2*)nullptr, ops->d_norms, ops->d_maxnorm, f->g_meta, (int*)nullptr,
              (int*)nullptr);
  PANO_LAUNCH(ctx, "k_tc_nominate", k_tc_pass<false>, std::min(max_blocks, ctx->num_sms), TC_THREADS, smem, f->gq, ops->tbuf, f->tasks,
              f->n_tasks, 0, ops->d_maxnorm, d_res, (const int*)nullptr, (int*)nullptr, (int*)nullptr);
  return PANO_OK;
}
