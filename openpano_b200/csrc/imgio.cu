// imgio.cu — the 8-bit image boundary either side of the hot path (SURVEY.md §8f.2-3):
//   read_img's u8 -> f32 conversion   (lib/imgio.cc:75-88)
//   crop()'s largest valid rectangle  (lib/imgproc.cc:200-235)
//   write_rgb's f32 -> u8 conversion  (lib/imgio.cc:98-113)
// so that 3 B/px cross PCIe instead of 12.  All three are HBM-bound byte movers.
#include "common.cuh"

// ------------------------------------------------------------------ u8 -> f32
struct Rgb8Job {
  const unsigned char* src;
  float* dst;
  long long n_px;
  int channels;   // the PANO_PIX_* format
  int pad;
};

// One CTA column per image (blockIdx.y); each thread converts 4 source bytes per
// trip.  The 256 possible quotients are built once per CTA with the reference's
// arithmetic — (float)((double)v / 255.0), imgio.cc:79-81 — and looked up.
__global__ void __launch_bounds__(256) k_rgb8_to_f32(const Rgb8Job* __restrict__ jobs) {
  __shared__ float lut[256];
  const Rgb8Job job = jobs[blockIdx.y];
  lut[threadIdx.x] = (float)((double)threadIdx.x / 255.0);
  __syncthreads();
  if (job.channels == 3) {
    const long long n = job.n_px * 3;
    const long long n4 = n >> 2;
    const uchar4* s4 = reinterpret_cast<const uchar4*>(job.src);
    float4* d4 = reinterpret_cast<float4*>(job.dst);
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4;
         i += (long long)gridDim.x * blockDim.x) {
      uchar4 v = __ldg(s4 + i);
      d4[i] = make_float4(lut[v.x], lut[v.y], lut[v.z], lut[v.w]);
    }
    if (blockIdx.x == 0 && threadIdx.x < (int)(n & 3)) {
      long long i = (n4 << 2) + threadIdx.x;
      job.dst[i] = lut[job.src[i]];
    }
  } else {
    // grey input: the value is replicated and NOT divided (imgio.cc:84-87)
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < job.n_px;
         i += (long long)gridDim.x * blockDim.x) {
      float v = (float)job.src[i];
      job.dst[i * 3 + 0] = v;
      job.dst[i * 3 + 1] = v;
      job.dst[i * 3 + 2] = v;
    }
  }
}

// The same for a batch that holds RGBA or planar images (any format per image), one pixel per thread and
// trip: RGBA (read_png, imgio.cc:43-61) is one 32-bit load whose fourth byte is ignored, planar (CImg,
// imgio.cc:72-88) reads the pixel's byte of each plane.  Every colour sample goes through the table except
// grey's, which is replicated undivided.
__global__ void __launch_bounds__(256) k_pix8_to_f32(const Rgb8Job* __restrict__ jobs) {
  __shared__ float lut[256];
  const Rgb8Job job = jobs[blockIdx.y];
  lut[threadIdx.x] = (float)((double)threadIdx.x / 255.0);
  __syncthreads();
  const unsigned char* src = job.src;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < job.n_px; i += (long long)gridDim.x * blockDim.x) {
    float r, g, b;
    if (job.channels == PANO_PIX_RGBA) {
      const unsigned t = __ldg(reinterpret_cast<const unsigned*>(src) + i);
      r = lut[t & 0xff]; g = lut[(t >> 8) & 0xff]; b = lut[(t >> 16) & 0xff];
    } else if (job.channels == PANO_PIX_RGB_PLANAR) {
      r = lut[__ldg(src + i)]; g = lut[__ldg(src + job.n_px + i)]; b = lut[__ldg(src + 2 * job.n_px + i)];
    } else if (job.channels == PANO_PIX_RGB) {
      r = lut[__ldg(src + 3 * i)]; g = lut[__ldg(src + 3 * i + 1)]; b = lut[__ldg(src + 3 * i + 2)];
    } else {
      r = g = b = (float)__ldg(src + i);
    }
    float* d = job.dst + i * 3;
    d[0] = r; d[1] = g; d[2] = b;
  }
}

// ------------------------------------------------------------------ crop rectangle
// The reference walks the lines top to bottom keeping, per column, the number of
// consecutive valid pixels ending at the line (`height`), and per line finds for
// every column the widest span whose heights are all >= its own (nearest strictly
// smaller neighbour either side).  The first maximum of span*height in
// (line, column) order wins (update_max is a strict >).
//
// Here: (1) one pass over the mosaic records a 32-line validity mask per column,
// (2) one CTA per line rebuilds that line's heights from the masks, finds the
// neighbours through a two-level min hierarchy in shared memory and reduces to the
// line's best, (3) one CTA reduces the lines.
//
// pano_crop_scan runs the same steps on each row strip of a mosaic: the masks are the
// strip's, the carry starts from the last invalid line of each column in the strips
// before (kept on the device), and (3) merges the strip's best into the best so far.
// Up to 40,000 columns its line kernel is (2) as is; wider lines, whose heights do not
// fit in shared memory, are read from the masks and the carry in global memory, so the
// width is not bounded by shared memory.

#define CROP_CHUNK 32

// std::max(a, b) is (a < b) ? b : a — kept literally so NaNs propagate as in the reference
__device__ __forceinline__ float std_max(float a, float b) { return (a < b) ? b : a; }

__global__ void __launch_bounds__(128) k_crop_masks(const float* __restrict__ mat, int w, int h,
                                                    unsigned* __restrict__ masks) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  const int c = blockIdx.y;
  if (k >= w) return;
  const int l0 = c * CROP_CHUNK;
  const int l1 = min(h, l0 + CROP_CHUNK);
  unsigned m = 0;
  for (int line = l0; line < l1; ++line) {
    const float* p = mat + ((size_t)line * w + k) * 3;
    float mx = std_max(std_max(p[0], p[1]), p[2]);
    if (mx < 0) m |= 1u << (line - l0);
  }
  masks[(size_t)c * w + k] = m;
}

struct CropLineBest {
  int area, k, left, right, height;
};

// carry[c][k] = last invalid line of column k in the chunks before c (-1 if none).  The masks
// start at line line0; last_io (null: -1 everywhere) holds each column's last invalid line before
// them and receives it after them.
__global__ void __launch_bounds__(128) k_crop_carry(const unsigned* __restrict__ masks, int w, int chunks, int line0,
                                                    int* __restrict__ last_io, int* __restrict__ carry) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= w) return;
  int last = last_io ? last_io[k] : -1;
  for (int c = 0; c < chunks; ++c) {
    carry[(size_t)c * w + k] = last;
    unsigned m = masks[(size_t)c * w + k];
    if (m) last = line0 + c * CROP_CHUNK + 31 - __clz(m);
  }
  if (last_io) last_io[k] = last;
}

#define CROP_RUN_CAP 2048
// Dynamic shared memory of k_crop_line<true>: the line's heights plus the run arrays (w <= 40,000 fits)
#define CROP_LINE_SMEM(w) (sizeof(int) * ((size_t)(w) + 4 * CROP_RUN_CAP + 1))
#define CROP_LINE_SMEM_MAX (200 * 1024)

// One CTA per line (line line0 + blockIdx.x of the mosaic, masks and carry as k_crop_carry
// leaves them).  kSmem: the line's heights are first copied to shared memory (w <= 40,000);
// otherwise every read recomputes a height from the masks and the carry.
// Columns of equal height that touch share their span, so the line
// is run-length encoded first (a mosaic line has a handful of runs: flat inside, a
// staircase at slanted borders) and the nearest-strictly-smaller neighbours are found
// per RUN by pointer jumping: l[r] starts at r-1 and hops to l[l[r]] while the run it
// points at is not lower — every hop keeps "all runs between l[r] and r are >= r", so
// any interleaving of the in-place updates is valid and the loop ends when a whole
// round changes nothing.  Lines with more than CROP_RUN_CAP runs take the per-column
// search through a two-level min hierarchy instead.
template <bool kSmem>
__global__ void __launch_bounds__(256) k_crop_line(const unsigned* __restrict__ masks, const int* __restrict__ carry,
                                                   int w, int line0, CropLineBest* __restrict__ best) {
  extern __shared__ int crop_smem[];
  int* hgt_s = crop_smem;                        // [w] (kSmem)
  int* r_start = hgt_s + (kSmem ? w : 0);        // [CAP + 1]   (fallback: l1, l2)
  int* r_h = r_start + CROP_RUN_CAP + 1;         // [CAP]
  int* r_l = r_h + CROP_RUN_CAP;                 // [CAP]
  int* r_r = r_l + CROP_RUN_CAP;                 // [CAP]
  __shared__ int s_warp[8];
  __shared__ unsigned long long s_key[8];
  __shared__ int s_pay[8][3];
  const int rel = blockIdx.x, line = line0 + rel;
  const int c = rel / CROP_CHUNK, bit = rel % CROP_CHUNK;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const unsigned* mrow = masks + (size_t)c * w;
  const int* crow = carry + (size_t)c * w;
  const unsigned lowmask = 0xFFFFFFFFu >> (31 - bit);
  // height of column k at `line`: lines since its last invalid line <= `line`
  auto hgt = [&](int k) -> int {
    if (kSmem) return hgt_s[k];
    const unsigned mm = __ldg(mrow + k) & lowmask;
    return line - (mm ? line0 + c * CROP_CHUNK + 31 - __clz(mm) : __ldg(crow + k));
  };

  if (kSmem) {
    // loads batched 8 deep (the loop is latency-bound otherwise)
    for (int k0 = tid; k0 < w; k0 += 8 * 256) {
      unsigned m[8];
      int cr[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        const int k = k0 + u * 256;
        m[u] = k < w ? __ldg(mrow + k) : 0u;
        cr[u] = k < w ? __ldg(crow + k) : 0;
      }
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        const int k = k0 + u * 256;
        if (k < w) {
          const unsigned mm = m[u] & lowmask;
          hgt_s[k] = line - (mm ? line0 + c * CROP_CHUNK + 31 - __clz(mm) : cr[u]);
        }
      }
    }
  }
  __syncthreads();

  // run starts: each thread owns an odd-length (bank-conflict-free) contiguous segment
  const int seg = ((w + 255) / 256) | 1;
  const int k0 = min(w, tid * seg), k1 = min(w, k0 + seg);
  int cnt = 0;
  for (int k = k0; k < k1; ++k) cnt += (k == 0 || hgt(k) != hgt(k - 1));
  int incl = cnt;
  for (int o = 1; o < 32; o <<= 1) {
    int v = __shfl_up_sync(0xFFFFFFFFu, incl, o);
    if (lane >= o) incl += v;
  }
  if (lane == 31) s_warp[warp] = incl;
  __syncthreads();
  int base = 0, total = 0;
  for (int i = 0; i < 8; ++i) { if (i < warp) base += s_warp[i]; total += s_warp[i]; }
  int off = base + incl - cnt;

  // key = (area, lowest column) packed so that a max picks the reference's winner
  unsigned long long key = 0;
  int b_left = 0, b_right = 0, b_h = 0;

  if (total <= CROP_RUN_CAP) {
    for (int k = k0; k < k1; ++k)
      if (k == 0 || hgt(k) != hgt(k - 1)) {
        r_start[off] = k; r_h[off] = hgt(k); r_l[off] = off - 1; r_r[off] = off + 1;
        ++off;
      }
    if (tid == 0) r_start[total] = w;
    __syncthreads();
    for (;;) {
      int ch = 0;
      for (int r = tid; r < total; r += blockDim.x) {
        const int v = r_h[r];
        int l = r_l[r];
        if (l >= 0 && r_h[l] >= v) { r_l[r] = r_l[l]; ch = 1; }
        int q = r_r[r];
        if (q < total && r_h[q] >= v) { r_r[r] = r_r[q]; ch = 1; }
      }
      if (!__syncthreads_or(ch)) break;
    }
    for (int r = tid; r < total; r += blockDim.x) {
      const int v = r_h[r];
      if (v == 0) continue;                    // area 0 never beats maxarea (strict >)
      const int left = r_start[r_l[r] + 1];
      const int right = r_start[r_r[r]] - 1;
      const int area = (right - left + 1) * v;
      const unsigned long long kk = ((unsigned long long)(unsigned)area << 32) | (0xFFFFFFFFu - (unsigned)r_start[r]);
      if (kk > key) { key = kk; b_left = left; b_right = right; b_h = v; }
    }
  } else {
    const int n1 = (w + 31) >> 5;
    const int n2 = (w + 1023) >> 10;
    int* l1 = r_start;                         // [n1] min over 32 columns
    int* l2 = l1 + n1;                         // [n2] min over 1024 columns
    for (int g = tid; g < n1; g += blockDim.x) {
      int mn = INT_MAX;
      const int e = min(w, (g + 1) << 5);
      for (int k = g << 5; k < e; ++k) mn = min(mn, hgt(k));
      l1[g] = mn;
    }
    __syncthreads();
    for (int g = tid; g < n2; g += blockDim.x) {
      int mn = INT_MAX;
      const int e = min(n1, (g + 1) << 5);
      for (int k = g << 5; k < e; ++k) mn = min(mn, l1[k]);
      l2[g] = mn;
    }
    __syncthreads();
    for (int k = tid; k < w; k += blockDim.x) {
      const int v = hgt(k);
      if (v == 0) continue;
      int j = k - 1;
      while (j >= 0) {
        if ((j & 1023) == 1023 && l2[j >> 10] >= v) { j -= 1024; continue; }
        if ((j & 31) == 31 && l1[j >> 5] >= v) { j -= 32; continue; }
        if (hgt(j) < v) break;
        --j;
      }
      const int left = j + 1;
      j = k + 1;
      while (j < w) {
        if ((j & 1023) == 0 && j + 1024 <= w && l2[j >> 10] >= v) { j += 1024; continue; }
        if ((j & 31) == 0 && j + 32 <= w && l1[j >> 5] >= v) { j += 32; continue; }
        if (hgt(j) < v) break;
        ++j;
      }
      const int right = j - 1;
      const int area = (right - left + 1) * v;
      const unsigned long long kk = ((unsigned long long)(unsigned)area << 32) | (0xFFFFFFFFu - (unsigned)k);
      if (kk > key) { key = kk; b_left = left; b_right = right; b_h = v; }
    }
  }
  // block arg-max
  for (int o = 16; o; o >>= 1) {
    unsigned long long ok = __shfl_down_sync(0xFFFFFFFFu, key, o);
    int ol = __shfl_down_sync(0xFFFFFFFFu, b_left, o);
    int orr = __shfl_down_sync(0xFFFFFFFFu, b_right, o);
    int oh = __shfl_down_sync(0xFFFFFFFFu, b_h, o);
    if (ok > key) { key = ok; b_left = ol; b_right = orr; b_h = oh; }
  }
  if (lane == 0) { s_key[warp] = key; s_pay[warp][0] = b_left; s_pay[warp][1] = b_right; s_pay[warp][2] = b_h; }
  __syncthreads();
  if (tid == 0) {
    int bw = 0;
    for (int i = 1; i < 8; ++i) if (s_key[i] > s_key[bw]) bw = i;
    CropLineBest r;
    r.area = (int)(s_key[bw] >> 32);
    r.k = (int)(0xFFFFFFFFu - (unsigned)(s_key[bw] & 0xFFFFFFFFu));
    r.left = s_pay[bw][0]; r.right = s_pay[bw][1]; r.height = s_pay[bw][2];
    best[rel] = r;
  }
}

// The best rectangle so far of a pano_crop_scan: area, last line, left and right column, height.
struct CropBest { int area, line, left, right, height; };

// Reduces the lines' bests (lines line0 + [0, h)) to crop()'s rectangle.  run (null: a whole
// mosaic) is the best of the lines above: this block's best replaces it only with a larger area,
// and the rectangle is the result.
__global__ void __launch_bounds__(256) k_crop_final(const CropLineBest* __restrict__ best, int h, int line0,
                                                    CropBest* __restrict__ run, int* __restrict__ rect) {
  unsigned long long key = 0;
  for (int line = threadIdx.x; line < h; line += blockDim.x) {
    int a = best[line].area;
    if (a > 0) {
      unsigned long long kk = ((unsigned long long)(unsigned)a << 32) | (0xFFFFFFFFu - (unsigned)line);
      if (kk > key) key = kk;
    }
  }
  __shared__ unsigned long long s_key[8];
  for (int o = 16; o; o >>= 1) {
    unsigned long long ok = __shfl_down_sync(0xFFFFFFFFu, key, o);
    if (ok > key) key = ok;
  }
  if ((threadIdx.x & 31) == 0) s_key[threadIdx.x >> 5] = key;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int i = 1; i < 8; ++i) if (s_key[i] > key) key = s_key[i];
    int ll = 0, rr = 0, hh = 0, nl = 0;            // crop()'s initial values (imgproc.cc:205)
    if (key) {
      const int q = (int)(0xFFFFFFFFu - (unsigned)(key & 0xFFFFFFFFu));
      nl = line0 + q;
      ll = best[q].left; rr = best[q].right; hh = best[q].height;
    }
    if (run) {
      if ((int)(key >> 32) > run->area) *run = CropBest{(int)(key >> 32), nl, ll, rr, hh};
      else { nl = run->line; ll = run->left; rr = run->right; hh = run->height; }
    }
    rect[0] = ll;                 // offsetx
    rect[1] = nl - hh + 1;        // offsety
    rect[2] = rr - ll + 1;        // width
    rect[3] = hh;                 // height
  }
}

// ------------------------------------------------------------------ f32 -> u8
// (v < 0 ? 1 : v) * 255 truncated to unsigned char (imgio.cc:107-109): Color::NO
// turns white.  One thread per output pixel of the (cropped) rectangle.
// The conversion is x86-64's: the float goes to int (f2i_x86), whose low byte is the sample.  A mosaic the caller
// hands in may hold anything: products in [256, 2^31) keep their low byte, and products >= 2^31, +inf and NaN give 0.
__global__ void __launch_bounds__(256) k_f32_to_rgb8(const float* __restrict__ mat, int w, int h,
                                                     const int* __restrict__ rect, unsigned char* __restrict__ out) {
  int x0 = 0, y0 = 0, cw = w, ch = h;
  if (rect) { x0 = rect[0]; y0 = rect[1]; cw = rect[2]; ch = rect[3]; }
  const long long n = (long long)cw * ch;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int r = (int)(i / cw), c = (int)(i - (long long)r * cw);
    const float* p = mat + ((size_t)(r + y0) * w + (c + x0)) * 3;
    unsigned char* o = out + i * 3;
#pragma unroll
    for (int q = 0; q < 3; ++q) {
      float v = p[q];
      v = (v < 0 ? 1.0f : v) * 255.0f;
      o[q] = (unsigned char)f2i_x86(v);
    }
  }
}

// k_f32_to_rgb8's samples in an encoder's layout: PANO_PIX_RGBA rows of 4 bytes per pixel with alpha 255
// (write_png, imgio.cc:25-41), or PANO_PIX_RGB_PLANAR, three planes of the rectangle's size (write_rgb's
// CImg<unsigned char>, imgio.cc:98-113).
template <int FMT>
__global__ void __launch_bounds__(256) k_f32_to_pix8(const float* __restrict__ mat, int w, int h,
                                                     const int* __restrict__ rect, unsigned char* __restrict__ out) {
  int x0 = 0, y0 = 0, cw = w, ch = h;
  if (rect) { x0 = rect[0]; y0 = rect[1]; cw = rect[2]; ch = rect[3]; }
  const long long n = (long long)cw * ch;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int r = (int)(i / cw), c = (int)(i - (long long)r * cw);
    const float* p = mat + ((size_t)(r + y0) * w + (c + x0)) * 3;
    unsigned char o[3];
#pragma unroll
    for (int q = 0; q < 3; ++q) {
      float v = p[q];
      v = (v < 0 ? 1.0f : v) * 255.0f;
      o[q] = (unsigned char)f2i_x86(v);
    }
    if (FMT == PANO_PIX_RGBA) {
      unsigned char* d = out + i * 4;
      d[0] = o[0]; d[1] = o[1]; d[2] = o[2]; d[3] = 255;
    } else {
      out[i] = o[0]; out[n + i] = o[1]; out[2 * n + i] = o[2];
    }
  }
}

// The crop rectangle of a mosaic converted by k_f32_to_rgb8 without a rect, in k_f32_to_pix8's layouts:
// the same bytes as converting the cropped f32 mosaic, since the conversion works sample by sample.
template <int FMT>
__global__ void __launch_bounds__(256) k_rgb8_crop(const unsigned char* __restrict__ rgb, int w, int h,
                                                   const int* __restrict__ rect, unsigned char* __restrict__ out) {
  int x0 = 0, y0 = 0, cw = w, ch = h;
  if (rect) { x0 = rect[0]; y0 = rect[1]; cw = rect[2]; ch = rect[3]; }
  const long long n = (long long)cw * ch;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int r = (int)(i / cw), c = (int)(i - (long long)r * cw);
    const unsigned char* p = rgb + ((size_t)(r + y0) * w + (c + x0)) * 3;
    const unsigned char o0 = p[0], o1 = p[1], o2 = p[2];
    if (FMT == PANO_PIX_RGBA) {
      unsigned char* d = out + i * 4;
      d[0] = o0; d[1] = o1; d[2] = o2; d[3] = 255;
    } else if (FMT == PANO_PIX_RGB_PLANAR) {
      out[i] = o0; out[n + i] = o1; out[2 * n + i] = o2;
    } else {
      unsigned char* d = out + i * 3;
      d[0] = o0; d[1] = o1; d[2] = o2;
    }
  }
}

// ------------------------------------------------------------------ crop scan state
#define CROP_SCAN_MAX_W 80000   // the reference's limit on a mosaic's edge (stitcher_image.cc:105)

struct pano_crop_scan {
  Sticky st;
  int w = 0, h = 0, lines = 0;
  DevBuf<int> d_last;        // [w] last invalid line of each column so far, -1 if none
  DevBuf<CropBest> d_run;    // the best rectangle so far
  DevBuf<int> d_rect;        // crop()'s rectangle of the lines so far
};

// Steps (1) to (3) on lines [line0, line0 + rows) of a w-column mosaic, d_strip holding those lines: d_last and d_run
// carry the lines before line0 (null for none), and d_rect gets crop()'s rectangle of the lines up to the last.
static int crop_strip(pano_ctx* ctx, const float* d_strip, int w, int rows, int line0, int* d_last, CropBest* d_run,
                      int* d_rect) {
  const int chunks = ceil_div(rows, CROP_CHUNK);
  DevBuf<unsigned> d_masks;
  DevBuf<int> d_carry;
  DevBuf<CropLineBest> d_best;
  int rc = 0;
  if ((rc = d_masks.alloc(ctx, (size_t)chunks * w)) || (rc = d_carry.alloc(ctx, (size_t)chunks * w)) ||
      (rc = d_best.alloc(ctx, (size_t)rows)))
    return rc;
  // the line kernel that keeps the line's heights in shared memory where they fit, else the one that reads them
  // from the masks and the carry (l1 / l2 of CROP_SCAN_MAX_W columns fit in the run arrays)
  const bool smem_line = CROP_LINE_SMEM(w) <= CROP_LINE_SMEM_MAX;
  const size_t smem = smem_line ? CROP_LINE_SMEM(w) : sizeof(int) * (4 * CROP_RUN_CAP + 1);
  if (smem_line && smem > 48 * 1024)
    PANO_CUDA(ctx, cudaFuncSetAttribute(k_crop_line<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  PANO_LAUNCH(ctx, "k_crop_masks", k_crop_masks, dim3(ceil_div(w, 128), chunks), 128, 0, d_strip, w, rows, d_masks);
  PANO_LAUNCH(ctx, "k_crop_carry", k_crop_carry, ceil_div(w, 128), 128, 0, d_masks, w, chunks, line0, d_last, d_carry);
  if (smem_line) PANO_LAUNCH(ctx, "k_crop_line", k_crop_line<true>, rows, 256, smem, d_masks, d_carry, w, line0, d_best);
  else PANO_LAUNCH(ctx, "k_crop_scan_line", k_crop_line<false>, rows, 256, smem, d_masks, d_carry, w, line0, d_best);
  PANO_LAUNCH(ctx, "k_crop_final", k_crop_final, 1, 256, 0, d_best, rows, line0, d_run, d_rect);
  return PANO_OK;
}

// ------------------------------------------------------------------ C API
extern "C" {

int pano_rgb8_to_mat32f_batch_dev(pano_ctx* ctx, int n, const unsigned char* const* d_pix, const int* w, const int* h,
                                  const int* channels, float* const* d_out_hwc) {
  ctx_enter(ctx);
  if (!ctx || n < 0 || (n && (!d_pix || !w || !h || !channels || !d_out_hwc)))
    return ctx_fail(ctx, PANO_ERR_INVALID, "pano_rgb8_to_mat32f_batch_dev: bad argument");
  if (n > PANO_MAX_IMAGES)   // images on gridDim.y
    return ctx_fail(ctx, PANO_ERR_INVALID, "pano_rgb8_to_mat32f_batch_dev: %d images in one batch (limit %d): split the batch",
                    n, PANO_MAX_IMAGES);
  if (n == 0) return PANO_OK;
  std::vector<Rgb8Job> jobs(n);
  long long max_px = 0;
  for (int i = 0; i < n; ++i) {
    if (w[i] <= 0 || h[i] <= 0 || !d_pix[i] || !d_out_hwc[i])
      return ctx_fail(ctx, PANO_ERR_INVALID, "pano_rgb8_to_mat32f_batch_dev: image %d: w=%d h=%d", i, w[i], h[i]);
    if (int rc = pix8_check(ctx, "pano_rgb8_to_mat32f_batch_dev", i, channels[i], d_pix[i])) return rc;
    if ((reinterpret_cast<uintptr_t>(d_pix[i]) & 3) || (reinterpret_cast<uintptr_t>(d_out_hwc[i]) & 15))
      return ctx_fail(ctx, PANO_ERR_INVALID, "pano_rgb8_to_mat32f_batch_dev: image %d: source must be 4-byte and "
                      "destination 16-byte aligned", i);
    jobs[i] = Rgb8Job{d_pix[i], d_out_hwc[i], (long long)w[i] * h[i], channels[i], 0};
    max_px = std::max(max_px, jobs[i].n_px);
  }
  DevBuf<Rgb8Job> d_jobs;
  if (int rc = d_jobs.alloc(ctx, n)) return rc;
  if (int rc = ctx_put(ctx, d_jobs, jobs.data(), sizeof(Rgb8Job) * n)) return rc;
  const bool layouts = src_reader(channels, n) == SrcReader::PIX8;   // an RGBA or planar image: k_pix8_to_f32
  long long per_img = ((layouts ? max_px : max_px * 3 / 4) + 255) / 256;
  int gx = (int)std::min<long long>(std::max<long long>(per_img, 1), std::max(1, ctx->num_sms * 8 / n));
  if (layouts) PANO_LAUNCH(ctx, "k_pix8_to_f32", k_pix8_to_f32, dim3(gx, n), 256, 0, d_jobs);
  else PANO_LAUNCH(ctx, "k_rgb8_to_f32", k_rgb8_to_f32, dim3(gx, n), 256, 0, d_jobs);
  return PANO_OK;
}

int pano_rgb8_to_mat32f_dev(pano_ctx* ctx, const unsigned char* d_pix, int w, int h, int channels, float* d_out_hwc) {
  ctx_enter(ctx);
  return pano_rgb8_to_mat32f_batch_dev(ctx, 1, &d_pix, &w, &h, &channels, &d_out_hwc);
}

int pano_crop_rect_dev(pano_ctx* ctx, const float* d_mat_hwc, int w, int h, int* d_rect) {
  ctx_enter(ctx);
  if (!ctx || !d_mat_hwc || !d_rect || w <= 0 || h <= 0)
    return ctx_fail(ctx, PANO_ERR_INVALID, "pano_crop_rect_dev: bad argument");
  // the widths whose line heights fit in shared memory: crop_strip's k_crop_line<true>
  if (CROP_LINE_SMEM(w) > CROP_LINE_SMEM_MAX)
    return ctx_fail(ctx, PANO_ERR_INVALID, "pano_crop_rect_dev: width %d exceeds the %d-column limit", w, 40000);
  return crop_strip(ctx, d_mat_hwc, w, h, 0, nullptr, nullptr, d_rect);
}

int pano_crop_scan_create(pano_ctx* ctx, int w, int h, pano_crop_scan** out) {
  ctx_enter(ctx);
  if (!ctx || !out) return PANO_ERR_INVALID;
  *out = nullptr;
  if (w <= 0 || h <= 0 || w > CROP_SCAN_MAX_W)
    return ctx_fail(ctx, PANO_ERR_INVALID, "crop scan: %dx%d (widths 1 to %d)", w, h, CROP_SCAN_MAX_W);
  std::unique_ptr<pano_crop_scan> c(new pano_crop_scan);
  c->st.ctx = ctx; c->w = w; c->h = h;
  int rc = 0;
  if ((rc = c->d_last.alloc(ctx, w)) || (rc = c->d_run.alloc(ctx, 1)) || (rc = c->d_rect.alloc(ctx, 4))) return rc;
  PANO_CUDA(ctx, cudaMemsetAsync(c->d_last, 0xff, sizeof(int) * w, ctx->stream));   // -1
  PANO_CUDA(ctx, cudaMemsetAsync(c->d_run, 0, sizeof(CropBest), ctx->stream));      // crop()'s initial values
  *out = c.release();
  return PANO_OK;
}

int pano_crop_scan_add_dev(pano_crop_scan* c, const float* d_strip_hwc, int rows) {
  if (!c) return PANO_ERR_INVALID;
  ctx_enter(c->st.ctx);
  if (c->st.err) return c->st.err;
  if (!d_strip_hwc || rows <= 0 || rows > c->h - c->lines)
    return c->st.misuse("crop scan: %d lines at line %d of %d", rows, c->lines, c->h);
  if (int rc = crop_strip(c->st.ctx, d_strip_hwc, c->w, rows, c->lines, c->d_last, c->d_run, c->d_rect))
    return c->st.fail(rc);
  c->lines += rows;
  return PANO_OK;
}

int pano_crop_scan_rect(pano_crop_scan* c, int rect[4]) {
  if (!c) return PANO_ERR_INVALID;
  pano_ctx* ctx = c->st.ctx;
  ctx_enter(ctx);
  if (c->st.err) return c->st.err;
  if (!rect) return c->st.misuse("crop scan: null rect");
  if (c->lines != c->h) return c->st.misuse("crop scan: rect after %d of %d lines", c->lines, c->h);
  cudaError_t e = cudaMemcpyAsync(rect, c->d_rect, 4 * sizeof(int), cudaMemcpyDeviceToHost, ctx->stream);
  if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
  return c->st.cuda(e, "crop scan: rect");
}

void pano_crop_scan_free(pano_crop_scan* c) {
  if (c) ctx_enter(c->st.ctx);
  delete c;
}

int pano_rgb8_crop_to_pix8_dev(pano_ctx* ctx, const unsigned char* d_rgb8, int w, int h, const int* d_rect, int format,
                               unsigned char* d_out) {
  ctx_enter(ctx);
  if (!ctx || !d_rgb8 || !d_out || w <= 0 || h <= 0)
    return ctx_fail(ctx, PANO_ERR_INVALID, "pano_rgb8_crop_to_pix8_dev: bad argument");
  long long blocks = ((long long)w * h + 255) / 256;
  int grid = (int)std::min<long long>(blocks, (long long)ctx->num_sms * 16);
  if (format == PANO_PIX_RGB)
    PANO_LAUNCH(ctx, "k_rgb8_crop", k_rgb8_crop<PANO_PIX_RGB>, grid, 256, 0, d_rgb8, w, h, d_rect, d_out);
  else if (format == PANO_PIX_RGBA)
    PANO_LAUNCH(ctx, "k_rgb8_crop_rgba", k_rgb8_crop<PANO_PIX_RGBA>, grid, 256, 0, d_rgb8, w, h, d_rect, d_out);
  else if (format == PANO_PIX_RGB_PLANAR)
    PANO_LAUNCH(ctx, "k_rgb8_crop_planar", k_rgb8_crop<PANO_PIX_RGB_PLANAR>, grid, 256, 0, d_rgb8, w, h, d_rect, d_out);
  else
    return ctx_fail(ctx, PANO_ERR_INVALID, "pano_rgb8_crop_to_pix8_dev: format %#x (PANO_PIX_RGB, _RGBA or _RGB_PLANAR)",
                    format);
  return PANO_OK;
}

int pano_mat32f_to_rgb8_dev(pano_ctx* ctx, const float* d_mat_hwc, int w, int h, const int* d_rect, unsigned char* d_out) {
  ctx_enter(ctx);
  if (!ctx || !d_mat_hwc || !d_out || w <= 0 || h <= 0)
    return ctx_fail(ctx, PANO_ERR_INVALID, "pano_mat32f_to_rgb8_dev: bad argument");
  long long blocks = ((long long)w * h + 255) / 256;
  int grid = (int)std::min<long long>(blocks, (long long)ctx->num_sms * 16);
  PANO_LAUNCH(ctx, "k_f32_to_rgb8", k_f32_to_rgb8, grid, 256, 0, d_mat_hwc, w, h, d_rect, d_out);
  return PANO_OK;
}

int pano_mat32f_to_pix8_dev(pano_ctx* ctx, const float* d_mat_hwc, int w, int h, const int* d_rect, int format,
                            unsigned char* d_out) {
  ctx_enter(ctx);
  if (!ctx || !d_mat_hwc || !d_out || w <= 0 || h <= 0)
    return ctx_fail(ctx, PANO_ERR_INVALID, "pano_mat32f_to_pix8_dev: bad argument");
  if (format == PANO_PIX_RGB) return pano_mat32f_to_rgb8_dev(ctx, d_mat_hwc, w, h, d_rect, d_out);
  if (format != PANO_PIX_RGBA && format != PANO_PIX_RGB_PLANAR)
    return ctx_fail(ctx, PANO_ERR_INVALID, "pano_mat32f_to_pix8_dev: format %#x (PANO_PIX_RGB, _RGBA or _RGB_PLANAR)", format);
  long long blocks = ((long long)w * h + 255) / 256;
  int grid = (int)std::min<long long>(blocks, (long long)ctx->num_sms * 16);
  if (format == PANO_PIX_RGBA)
    PANO_LAUNCH(ctx, "k_f32_to_rgba8", k_f32_to_pix8<PANO_PIX_RGBA>, grid, 256, 0, d_mat_hwc, w, h, d_rect, d_out);
  else
    PANO_LAUNCH(ctx, "k_f32_to_planar8", k_f32_to_pix8<PANO_PIX_RGB_PLANAR>, grid, 256, 0, d_mat_hwc, w, h, d_rect, d_out);
  return PANO_OK;
}

}  // extern "C"
