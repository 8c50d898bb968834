// motionseg.cu -- moving-object segmentation: a per-pixel score of camera-relative motion, thresholded with hysteresis and
// labelled into 8-connected objects with per-object statistics.
//
//   mfn_motion_segment   residuals and occlusion masks of both flow directions on each frame (mfn_affine_motion's
//                        residual, mfn_flow_consistency's masks), side a's flow and affine fit
//                        ->  labels (N,H,W) uint8, objects (N,max_objects,10) float64, count (N), dropped (N)
//     every launch has grid y = N, one frame per grid row; 11 launches whatever the content (the rule is in
//     include/maskflow_b200.h):
//       seg_init_kernel      one thread per pixel: the score s, computed inline; parent[p] = p where s >= tau_lo, else -1
//       seg_merge_kernel     one thread per pixel: union with the foreground neighbours W, NW, N, NE (Playne and Hawick,
//                            IEEE TPDS 2018): the larger root is linked under the smaller with atomicMin, so
//                            parent[i] <= i always holds and every root ends as its component's first pixel
//       seg_count_kernel     per 4096-pixel tile: path compression of each pixel, the number of roots in the tile
//       seg_scan_kernel      per frame: exclusive scan of the tile counts (the first pass of a multi-CTA scan)
//       seg_number_kernel    per tile: each root gets its compact id, tile offset + rank in the tile, stored in its parent
//                            slot as -2 - id; its statistics are cleared
//       seg_stats_kernel     per tile: area and peak s per compact id, integer atomics once per run of equal ids
//       seg_keep_kernel      per tile of 4096 ids: how many components are kept (area >= min_area, peak >= tau_hi)
//       seg_scan_kernel      per frame: exclusive scan of those counts; count and dropped; the object sums are cleared
//       seg_assign_kernel    per tile of ids: kept component of rank r gets label r + 1 (0 past max_objects)
//       seg_label_kernel     per tile: labels, and per object the box, the coordinate sums and the fixed-point
//                            displacement sums, integer atomics once per run of equal labels
//       seg_objects_kernel   per frame: the object rows
//     Integer atomics only, and the labels do not depend on the order of the unions: bit-reproducible.  No allocation,
//     no host synchronisation, a launch configuration that depends on the extents only: capture-safe.
//
// The file also builds for the host (MFN_HOST_EMULATION: tests/host_emu/motionseg_emu.cpp).  The kernels are composed of
// per-thread device functions; the tile kernels' block scans and reductions are done by the emulation in between, and
// there every step of a find asserts parent[i] < i.
#ifdef MFN_HOST_EMULATION
#include <cassert>

#include "cuda_shim.h"
#define SEG_ASSERT(c) assert(c)
#else
#include <math.h>

#include "common.cuh"
#define SEG_ASSERT(c) ((void)0)
#endif

namespace mfn {

constexpr int kSegThreads = 256;                       // threads of every per-pixel and per-tile kernel
constexpr int kSegRun = 16;                            // contiguous pixels (or ids) per thread in the tile kernels
constexpr int kSegTile = kSegThreads * kSegRun;        // 4096
constexpr int kSegScanThreads = 1024;
constexpr int kSegMaxObjects = 255;
constexpr int kSegObjCols = 10;
constexpr double kSegClamp = 65536.0;                  // |displacement| is clamped to 2^16 px before it is summed

// One kept object's sums.  Signed sums are added as two's complement unsigned 64-bit integers.
struct SegAcc {
  unsigned long long sx, sy;       // sum of x, sum of y over the object's pixels
  unsigned long long dx, dy;       // sum of rint(d 2^S) over the pixels where side a is defined (two's complement)
  int x0, y0, x1, y1;
  unsigned area, peak, na, pad;    // peak: seg_key of the largest score
};

// Extents of the workspace: per frame HW parents, T1 tile counts, C compact components (area, peak key, label), T2 tile
// counts of kept components, 2 totals, 255 object sums.
struct SegLayout {
  long long HW, C, T1, T2;
  long long off_parent, off_tiles, off_ktiles, off_comp, off_tot, off_acc, bytes;
};

__host__ __device__ inline long long seg_align(long long v) { return (v + 255) & ~255LL; }

__host__ __device__ inline SegLayout seg_layout(int N, int H, int W) {
  SegLayout s;
  s.HW = (long long)H * W;
  s.C = (long long)((H + 1) / 2) * ((W + 1) / 2);   // every 2x2 block meets at most one 8-connected component
  s.T1 = (s.HW + kSegTile - 1) / kSegTile;
  s.T2 = (s.C + kSegTile - 1) / kSegTile;
  long long o = 0;
  s.off_parent = o, o = seg_align(o + 4 * N * s.HW);
  s.off_tiles = o, o = seg_align(o + 4 * N * s.T1);
  s.off_ktiles = o, o = seg_align(o + 4 * N * s.T2);
  s.off_comp = o, o = seg_align(o + 12 * N * s.C);
  s.off_tot = o, o = seg_align(o + 8 * (long long)N);
  s.off_acc = o, o = seg_align(o + (long long)sizeof(SegAcc) * kSegMaxObjects * N);
  s.bytes = o;
  return s;
}

// S: the displacement's fixed-point scale 2^S, S = 46 - k with 2^(k-1) <= HW < 2^k, so that HW terms of at most
// 2^16 2^S each add to less than 2^62.
__host__ __device__ inline int seg_scale_bits(long long HW) {
  int k = 0;
  while ((1LL << k) <= HW) ++k;
  return 46 - k;
}

// Order-preserving key of a float: keys compare as unsigned integers like the floats they encode (-0 below +0).
__device__ __forceinline__ unsigned seg_key(float v) {
  const unsigned b = __float_as_uint(v);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float seg_unkey(unsigned k) {
  const unsigned b = (k & 0x80000000u) ? (k & 0x7fffffffu) : ~k;
  return __uint_as_float(b);
}

// s at pixel i: the smaller of the defined residuals of the two sides, NaN where neither is defined
__device__ __forceinline__ float seg_score(const float* __restrict__ res_a, const unsigned char* __restrict__ occ_a,
                                           const float* __restrict__ res_b, const unsigned char* __restrict__ occ_b,
                                           size_t i) {
  float s = __int_as_float(0x7fc00000);
  bool def = false;
  if (res_a) {
    const float a = __ldg(res_a + i);
    if (isfinite(a) && __ldg(occ_a + i) == 0) s = a, def = true;
  }
  if (res_b) {
    const float b = __ldg(res_b + i);
    if (isfinite(b) && __ldg(occ_b + i) == 0) s = def ? fminf(s, b) : b;
  }
  return s;
}

__device__ __forceinline__ int seg_load(const int* p) {
#ifdef MFN_HOST_EMULATION
  return *(const volatile int*)p;
#else
  return __ldcg(p);   // at L2, where the atomics are: no stale L1 copy
#endif
}

// The root of x, halving the path on the way with atomicMin (a parent only ever decreases, towards an ancestor).
__device__ __forceinline__ int seg_find(int* L, int x) {
  int v = seg_load(L + x);
  while (v != x) {
    SEG_ASSERT(v >= 0 && v < x);
    const int w = seg_load(L + v);
    SEG_ASSERT(w >= 0 && w <= v);
    if (w != v) atomicMin(L + x, w);
    x = v;
    v = w;
  }
  return x;
}

// Links the trees of a and b: the larger root under the smaller.  When the root was linked meanwhile, atomicMin returns
// its new parent and the union goes on from there.
__device__ __forceinline__ void seg_union(int* L, int a, int b) {
  for (;;) {
    a = seg_find(L, a);
    b = seg_find(L, b);
    if (a == b) return;
    if (a > b) {
      const int t = a;
      a = b;
      b = t;
    }
    const int old = atomicMin(L + b, a);
    SEG_ASSERT(old <= b);
    if (old == b) return;
    b = old;
  }
}

// ---- per-pixel phases: pixel p of frame n, i = n HW + p ---------------------------------------------------------------
__device__ __forceinline__ void seg_init_pixel(const float* __restrict__ res_a, const unsigned char* __restrict__ occ_a,
                                               const float* __restrict__ res_b, const unsigned char* __restrict__ occ_b,
                                               int* __restrict__ L, int HW, int n, int p, float tau_lo) {
  const size_t i = (size_t)n * HW + p;
  L[i] = seg_score(res_a, occ_a, res_b, occ_b, i) >= tau_lo ? p : -1;
}

__device__ __forceinline__ void seg_merge_pixel(int* L, int H, int W, int p) {
  if (seg_load(L + p) < 0) return;
  const int y = p / W, x = p - y * W;
  if (x > 0 && seg_load(L + p - 1) >= 0) seg_union(L, p, p - 1);
  if (y > 0) {
    const int q = p - W;
    if (x > 0 && seg_load(L + q - 1) >= 0) seg_union(L, p, q - 1);
    if (seg_load(L + q) >= 0) seg_union(L, p, q);
    if (x + 1 < W && seg_load(L + q + 1) >= 0) seg_union(L, p, q + 1);
  }
}

// ---- tile phases: thread t of tile g owns the items [g 4096 + 16 t, + 16) -------------------------------------------
__device__ __forceinline__ void seg_range(int g, int t, long long n, int* b, int* e) {
  const long long b0 = (long long)g * kSegTile + (long long)t * kSegRun;
  *b = (int)(b0 < n ? b0 : n);
  *e = (int)(b0 + kSegRun < n ? b0 + kSegRun : n);
}

// path compression of the thread's pixels (frame-local L); returns how many of them are roots
__device__ __forceinline__ int seg_compress_count(int* L, int HW, int g, int t) {
  int b, e, c = 0;
  seg_range(g, t, HW, &b, &e);
  for (int p = b; p < e; ++p) {
    if (L[p] < 0) continue;
    const int r = seg_find(L, p);
    L[p] = r;
    c += r == p;
  }
  return c;
}

__device__ __forceinline__ int seg_count_roots(const int* L, int HW, int g, int t) {
  int b, e, c = 0;
  seg_range(g, t, HW, &b, &e);
  for (int p = b; p < e; ++p) c += L[p] == p;
  return c;
}

// roots get the ids id0, id0 + 1, ... in pixel order; comp (C,3): area, peak key, label
__device__ __forceinline__ void seg_number_roots(int* L, unsigned* comp, int HW, int g, int t, int id0) {
  int b, e;
  seg_range(g, t, HW, &b, &e);
  for (int p = b; p < e; ++p) {
    if (L[p] != p) continue;
    L[p] = -2 - id0;
    comp[3 * (size_t)id0] = 0;
    comp[3 * (size_t)id0 + 1] = 0;
    comp[3 * (size_t)id0 + 2] = 0;
    ++id0;
  }
}

// the compact id of foreground pixel p (after seg_number_roots), -1 for the background
__device__ __forceinline__ int seg_id(const int* L, int p) {
  const int v = L[p];
  if (v == -1) return -1;
  return v <= -2 ? -2 - v : -2 - L[v];
}

__device__ __forceinline__ void seg_stats_run(const float* __restrict__ res_a, const unsigned char* __restrict__ occ_a,
                                              const float* __restrict__ res_b, const unsigned char* __restrict__ occ_b,
                                              const int* L, unsigned* comp, int HW, int n, int g, int t) {
  int b, e;
  seg_range(g, t, HW, &b, &e);
  int cur = -1;
  unsigned area = 0, peak = 0;
  for (int p = b; p <= e; ++p) {
    const int c = p < e ? seg_id(L, p) : -1;
    if (c != cur && cur >= 0) {
      atomicAdd(comp + 3 * (size_t)cur, area);
      atomicMax(comp + 3 * (size_t)cur + 1, peak);
    }
    if (c < 0) {
      cur = -1;
      continue;
    }
    const unsigned k = seg_key(seg_score(res_a, occ_a, res_b, occ_b, (size_t)n * HW + p));
    if (c != cur) {
      cur = c, area = 1, peak = k;
    } else {
      ++area;
      peak = k > peak ? k : peak;
    }
  }
}

__device__ __forceinline__ bool seg_kept(const unsigned* comp, int c, int min_area, float tau_hi) {
  return comp[3 * (size_t)c] >= (unsigned)min_area && seg_unkey(comp[3 * (size_t)c + 1]) >= tau_hi;
}

__device__ __forceinline__ int seg_count_kept(const unsigned* comp, int R, int g, int t, int min_area, float tau_hi) {
  int b, e, k = 0;
  seg_range(g, t, R, &b, &e);
  for (int c = b; c < e; ++c) k += seg_kept(comp, c, min_area, tau_hi);
  return k;
}

// kept components of rank r0, r0 + 1, ... in id order: label r + 1 up to max_objects, and the object's area and peak
__device__ __forceinline__ void seg_assign(unsigned* comp, SegAcc* acc, int R, int g, int t, int r0, int min_area,
                                           float tau_hi, int max_objects) {
  int b, e;
  seg_range(g, t, R, &b, &e);
  for (int c = b; c < e; ++c) {
    unsigned lab = 0;
    if (seg_kept(comp, c, min_area, tau_hi)) {
      if (r0 < max_objects) {
        lab = (unsigned)r0 + 1;
        acc[r0].area = comp[3 * (size_t)c];
        acc[r0].peak = comp[3 * (size_t)c + 1];
      }
      ++r0;
    }
    comp[3 * (size_t)c + 2] = lab;
  }
}

// after the scan of the kept counts: the frame's count and dropped, and the object sums cleared
__device__ __forceinline__ void seg_clear_objects(SegAcc* acc, int t, int T, int kept, int max_objects, int* count,
                                                  int* dropped) {
  for (int j = t; j < max_objects; j += T) {
    SegAcc& a = acc[j];
    a.sx = a.sy = a.dx = a.dy = 0;
    a.x0 = a.y0 = 0x7fffffff;
    a.x1 = a.y1 = -1;
    a.area = a.peak = a.na = a.pad = 0;
  }
  if (t == 0) {
    *count = kept < max_objects ? kept : max_objects;
    *dropped = kept > max_objects ? kept - max_objects : 0;
  }
}

// d = (p + flow(p)) - A p along one axis, each operation rounded on its own (no contraction), clamped to +-2^16 px
__device__ __forceinline__ double seg_disp(double pxy, float u, double a0, double a1, double a2, double x, double y) {
  const double q = __dadd_rn(pxy, (double)u);
  const double m = __dadd_rn(__dadd_rn(__dmul_rn(a0, x), __dmul_rn(a1, y)), a2);
  const double d = __dsub_rn(q, m);
  return fmin(fmax(d, -kSegClamp), kSegClamp);
}

struct SegRun {
  unsigned long long sx, sy, dx, dy;
  int x0, y0, x1, y1;
  unsigned na;
};

__device__ __forceinline__ void seg_flush(SegAcc* a, const SegRun& r) {
  atomicAdd(&a->sx, r.sx);
  atomicAdd(&a->sy, r.sy);
  if (r.na) {
    atomicAdd(&a->dx, r.dx);
    atomicAdd(&a->dy, r.dy);
    atomicAdd(&a->na, r.na);
  }
  atomicMin(&a->x0, r.x0);
  atomicMin(&a->y0, r.y0);
  atomicMax(&a->x1, r.x1);
  atomicMax(&a->y1, r.y1);
}

__device__ __forceinline__ void seg_label_run(const float* __restrict__ res_a, const unsigned char* __restrict__ occ_a,
                                              const float2* __restrict__ flow_a, const double* __restrict__ affine_a,
                                              const int* L, const unsigned* comp, SegAcc* acc,
                                              unsigned char* __restrict__ labels, int W, int HW, int n, int g, int t,
                                              int S) {
  int b, e;
  seg_range(g, t, HW, &b, &e);
  const double scale = ldexp(1.0, S);
  double a[6] = {0, 0, 0, 0, 0, 0};
  if (affine_a)
    for (int k = 0; k < 6; ++k) a[k] = affine_a[6 * (size_t)n + k];
  int cur = 0;
  SegRun r = {};
  for (int p = b; p <= e; ++p) {
    int lab = 0;
    if (p < e) {
      const int c = seg_id(L, p);
      lab = c < 0 ? 0 : (int)comp[3 * (size_t)c + 2];
      labels[(size_t)n * HW + p] = (unsigned char)lab;
    }
    if (lab != cur) {   // a run of equal labels ends: its sums go to the object with one atomic each
      if (cur > 0) seg_flush(acc + cur - 1, r);
      cur = lab;
      r = SegRun{0, 0, 0, 0, 0x7fffffff, 0x7fffffff, -1, -1, 0};
    }
    if (lab == 0) continue;
    const int y = p / W, x = p - y * W;
    r.sx += (unsigned long long)x;
    r.sy += (unsigned long long)y;
    r.x0 = min(r.x0, x), r.y0 = min(r.y0, y), r.x1 = max(r.x1, x), r.y1 = max(r.y1, y);
    if (res_a) {
      const size_t i = (size_t)n * HW + p;
      const float ra = __ldg(res_a + i);
      if (isfinite(ra) && __ldg(occ_a + i) == 0) {
        const float2 uv = __ldg(flow_a + i);
        const double xd = (double)x, yd = (double)y;
        r.dx += (unsigned long long)llrint(seg_disp(xd, uv.x, a[0], a[1], a[2], xd, yd) * scale);
        r.dy += (unsigned long long)llrint(seg_disp(yd, uv.y, a[3], a[4], a[5], xd, yd) * scale);
        ++r.na;
      }
    }
  }
}

__device__ __forceinline__ void seg_object_row(const SegAcc& a, int j, int count, int S, double* __restrict__ row) {
  if (j >= count) {
    for (int k = 0; k < kSegObjCols; ++k) row[k] = 0.0;
    return;
  }
  const double area = (double)a.area;
  row[0] = area;
  row[1] = (double)a.x0, row[2] = (double)a.y0, row[3] = (double)a.x1, row[4] = (double)a.y1;
  row[5] = (double)a.sx / area;
  row[6] = (double)a.sy / area;
  row[7] = (double)seg_unkey(a.peak);
  if (a.na == 0) {
    row[8] = row[9] = __longlong_as_double(0x7ff8000000000000LL);
  } else {
    const double inv = ldexp(1.0, -S);
    row[8] = (double)(long long)a.dx * inv / (double)a.na;
    row[9] = (double)(long long)a.dy * inv / (double)a.na;
  }
}

#ifndef MFN_HOST_EMULATION
// exclusive scan of v over the CTA; *total = the sum.  Every thread of the CTA must call it.
__device__ __forceinline__ int seg_block_scan(int v, int* total) {
  __shared__ int warp_sum[32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarp = blockDim.x >> 5;
  int x = v;
  for (int o = 1; o < 32; o <<= 1) {
    const int y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) warp_sum[warp] = x;
  __syncthreads();
  if (warp == 0) {
    int w = lane < nwarp ? warp_sum[lane] : 0;
    for (int o = 1; o < 32; o <<= 1) {
      const int y = __shfl_up_sync(0xffffffffu, w, o);
      if (lane >= o) w += y;
    }
    if (lane < nwarp) warp_sum[lane] = w;
  }
  __syncthreads();
  const int excl = x - v + (warp > 0 ? warp_sum[warp - 1] : 0);
  *total = warp_sum[nwarp - 1];
  __syncthreads();   // warp_sum is reused by the next call
  return excl;
}

struct SegPtrs {
  int* parent;        // (N, HW)
  int* tiles;         // (N, T1)
  int* ktiles;        // (N, T2)
  unsigned* comp;     // (N, C, 3)
  int* tot;           // (N, 2): roots, kept components
  SegAcc* acc;        // (N, 255)
};

// grid (ceil(HW / 256), N)
__global__ void __launch_bounds__(kSegThreads)
    seg_init_kernel(const float* __restrict__ res_a, const unsigned char* __restrict__ occ_a,
                    const float* __restrict__ res_b, const unsigned char* __restrict__ occ_b, int* __restrict__ parent,
                    int HW, float tau_lo) {
  const int p = blockIdx.x * kSegThreads + threadIdx.x;
  if (p < HW) seg_init_pixel(res_a, occ_a, res_b, occ_b, parent, HW, blockIdx.y, p, tau_lo);
}

// grid (ceil(HW / 256), N)
__global__ void __launch_bounds__(kSegThreads) seg_merge_kernel(int* parent, int H, int W) {
  const int HW = H * W;
  const int p = blockIdx.x * kSegThreads + threadIdx.x;
  if (p < HW) seg_merge_pixel(parent + (size_t)blockIdx.y * HW, H, W, p);
}

// grid (T1, N)
__global__ void __launch_bounds__(kSegThreads) seg_count_kernel(SegPtrs w, int HW, int T1) {
  const int n = blockIdx.y, g = blockIdx.x;
  const int c = seg_compress_count(w.parent + (size_t)n * HW, HW, g, threadIdx.x);
  int total;
  seg_block_scan(c, &total);
  if (threadIdx.x == 0) w.tiles[(size_t)n * T1 + g] = total;
}

// grid N, 1024 threads: exclusive scan of counts (N, T) in place, tot[n * 2 + which] = the sum; which == 1 also
// finishes the frame's count and dropped and clears its object sums
__global__ void __launch_bounds__(kSegScanThreads)
    seg_scan_kernel(int* __restrict__ counts, int T, int* __restrict__ tot, int which, SegAcc* __restrict__ acc,
                    int max_objects, int* __restrict__ count, int* __restrict__ dropped) {
  const int n = blockIdx.x, t = threadIdx.x;
  int* c = counts + (size_t)n * T;
  const int chunk = (T + kSegScanThreads - 1) / kSegScanThreads;
  const int b = min(t * chunk, T), e = min(b + chunk, T);
  int sum = 0;
  for (int i = b; i < e; ++i) sum += c[i];
  int total;
  int run = seg_block_scan(sum, &total);
  for (int i = b; i < e; ++i) {
    const int v = c[i];
    c[i] = run;
    run += v;
  }
  if (t == 0) tot[2 * n + which] = total;
  if (which == 1) seg_clear_objects(acc + (size_t)n * kSegMaxObjects, t, kSegScanThreads, total, max_objects, count + n,
                                    dropped + n);
}

// grid (T1, N)
__global__ void __launch_bounds__(kSegThreads) seg_number_kernel(SegPtrs w, int HW, int T1, long long C) {
  const int n = blockIdx.y, g = blockIdx.x;
  int* L = w.parent + (size_t)n * HW;
  int total;
  const int r = seg_block_scan(seg_count_roots(L, HW, g, threadIdx.x), &total);
  seg_number_roots(L, w.comp + (size_t)n * C * 3, HW, g, threadIdx.x, w.tiles[(size_t)n * T1 + g] + r);
}

// grid (T1, N)
__global__ void __launch_bounds__(kSegThreads)
    seg_stats_kernel(const float* __restrict__ res_a, const unsigned char* __restrict__ occ_a,
                     const float* __restrict__ res_b, const unsigned char* __restrict__ occ_b, SegPtrs w, int HW,
                     long long C) {
  const int n = blockIdx.y;
  seg_stats_run(res_a, occ_a, res_b, occ_b, w.parent + (size_t)n * HW, w.comp + (size_t)n * C * 3, HW, n, blockIdx.x,
                threadIdx.x);
}

// grid (T2, N)
__global__ void __launch_bounds__(kSegThreads)
    seg_keep_kernel(SegPtrs w, long long C, int T2, int min_area, float tau_hi) {
  const int n = blockIdx.y, g = blockIdx.x;
  const int R = w.tot[2 * n];
  int total;
  seg_block_scan(seg_count_kept(w.comp + (size_t)n * C * 3, R, g, threadIdx.x, min_area, tau_hi), &total);
  if (threadIdx.x == 0) w.ktiles[(size_t)n * T2 + g] = total;
}

// grid (T2, N)
__global__ void __launch_bounds__(kSegThreads)
    seg_assign_kernel(SegPtrs w, long long C, int T2, int min_area, float tau_hi, int max_objects) {
  const int n = blockIdx.y, g = blockIdx.x;
  const int R = w.tot[2 * n];
  unsigned* comp = w.comp + (size_t)n * C * 3;
  int total;
  const int r = seg_block_scan(seg_count_kept(comp, R, g, threadIdx.x, min_area, tau_hi), &total);
  seg_assign(comp, w.acc + (size_t)n * kSegMaxObjects, R, g, threadIdx.x, w.ktiles[(size_t)n * T2 + g] + r, min_area,
             tau_hi, max_objects);
}

// grid (T1, N)
__global__ void __launch_bounds__(kSegThreads)
    seg_label_kernel(const float* __restrict__ res_a, const unsigned char* __restrict__ occ_a,
                     const float2* __restrict__ flow_a, const double* __restrict__ affine_a, SegPtrs w,
                     unsigned char* __restrict__ labels, int W, int HW, long long C, int S) {
  const int n = blockIdx.y;
  seg_label_run(res_a, occ_a, flow_a, affine_a, w.parent + (size_t)n * HW, w.comp + (size_t)n * C * 3,
                w.acc + (size_t)n * kSegMaxObjects, labels, W, HW, n, blockIdx.x, threadIdx.x, S);
}

// grid N, 256 threads: row j of frame n
__global__ void __launch_bounds__(kSegThreads)
    seg_objects_kernel(const SegAcc* __restrict__ acc, const int* __restrict__ count, double* __restrict__ objects,
                       int max_objects, int S) {
  const int n = blockIdx.x, j = threadIdx.x;
  if (j >= max_objects) return;
  seg_object_row(acc[(size_t)n * kSegMaxObjects + j], j, count[n], S,
                 objects + ((size_t)n * max_objects + j) * kSegObjCols);
}
#endif  // !MFN_HOST_EMULATION

}  // namespace mfn

#ifndef MFN_HOST_EMULATION
extern "C" long long mfn_motion_segment_workspace_bytes(int N, int H, int W) {
  return (N > 0 && H > 0 && W > 0) ? mfn::seg_layout(N, H, W).bytes : 0;
}

extern "C" int mfn_motion_segment(const float* res_a, const unsigned char* occ_a, const float* res_b,
                                  const unsigned char* occ_b, const float* flow_a, const double* affine_a,
                                  unsigned char* labels, double* objects, int* count, int* dropped, void* ws,
                                  long long ws_bytes, int N, int H, int W, float tau_lo, float tau_hi, int min_area,
                                  int max_objects, void* stream) {
  using namespace mfn;
  const bool side_a = res_a || occ_a || flow_a || affine_a, side_b = res_b || occ_b;
  MFN_REQUIRE(labels && objects && count && dropped && ws, MFN_ERR_INVALID_ARG, "mfn_motion_segment: null pointer");
  MFN_REQUIRE(!side_a || (res_a && occ_a && flow_a && affine_a), MFN_ERR_INVALID_ARG,
              "mfn_motion_segment: null pointer: res_a, occ_a, flow_a and affine_a go together");
  MFN_REQUIRE(!side_b || (res_b && occ_b), MFN_ERR_INVALID_ARG,
              "mfn_motion_segment: null pointer: res_b and occ_b go together");
  MFN_REQUIRE(N > 0 && H > 0 && W > 0, MFN_ERR_INVALID_ARG, "mfn_motion_segment: non-positive extent");
  MFN_REQUIRE(isfinite(tau_lo) && isfinite(tau_hi) && tau_lo <= tau_hi, MFN_ERR_INVALID_ARG,
              "mfn_motion_segment: tau_lo and tau_hi must be finite with tau_lo <= tau_hi, got %g, %g", (double)tau_lo,
              (double)tau_hi);
  MFN_REQUIRE(min_area >= 1, MFN_ERR_INVALID_ARG, "mfn_motion_segment: min_area must be >= 1, got %d", min_area);
  MFN_REQUIRE(max_objects >= 1 && max_objects <= kSegMaxObjects, MFN_ERR_INVALID_ARG,
              "mfn_motion_segment: max_objects must lie in [1,255], got %d", max_objects);
  MFN_REQUIRE(aligned(res_a, 4) && aligned(res_b, 4) && aligned(flow_a, 8) && aligned(affine_a, 8) &&
                  aligned(objects, 8) && aligned(count, 4) && aligned(dropped, 4) && aligned(ws, 16),
              MFN_ERR_INVALID_ARG,
              "mfn_motion_segment: res_a, res_b, count and dropped must be 4-byte aligned, flow_a, affine_a and objects "
              "8-byte, ws 16-byte");
  MFN_REQUIRE((long long)H * W < (1LL << 31) && N <= 65535, MFN_ERR_ALIGNMENT,
              "mfn_motion_segment: extents overflow kernel indexing");
  const SegLayout lay = seg_layout(N, H, W);
  MFN_REQUIRE(ws_bytes >= lay.bytes, MFN_ERR_INVALID_ARG, "mfn_motion_segment: workspace of %lld bytes, %lld needed",
              ws_bytes, lay.bytes);
  char* base = static_cast<char*>(ws);
  SegPtrs w;
  w.parent = reinterpret_cast<int*>(base + lay.off_parent);
  w.tiles = reinterpret_cast<int*>(base + lay.off_tiles);
  w.ktiles = reinterpret_cast<int*>(base + lay.off_ktiles);
  w.comp = reinterpret_cast<unsigned*>(base + lay.off_comp);
  w.tot = reinterpret_cast<int*>(base + lay.off_tot);
  w.acc = reinterpret_cast<SegAcc*>(base + lay.off_acc);
  const int HW = H * W, T1 = (int)lay.T1, T2 = (int)lay.T2, S = seg_scale_bits(lay.HW);
  const dim3 px((HW + kSegThreads - 1) / kSegThreads, N), tiles(T1, N), ids(T2, N);
  cudaStream_t st = as_stream(stream);
  seg_init_kernel<<<px, kSegThreads, 0, st>>>(res_a, occ_a, res_b, occ_b, w.parent, HW, tau_lo);
  if (int rc = check_launch("seg_init_kernel")) return rc;
  seg_merge_kernel<<<px, kSegThreads, 0, st>>>(w.parent, H, W);
  if (int rc = check_launch("seg_merge_kernel")) return rc;
  seg_count_kernel<<<tiles, kSegThreads, 0, st>>>(w, HW, T1);
  if (int rc = check_launch("seg_count_kernel")) return rc;
  seg_scan_kernel<<<N, kSegScanThreads, 0, st>>>(w.tiles, T1, w.tot, 0, w.acc, max_objects, count, dropped);
  if (int rc = check_launch("seg_scan_kernel")) return rc;
  seg_number_kernel<<<tiles, kSegThreads, 0, st>>>(w, HW, T1, lay.C);
  if (int rc = check_launch("seg_number_kernel")) return rc;
  seg_stats_kernel<<<tiles, kSegThreads, 0, st>>>(res_a, occ_a, res_b, occ_b, w, HW, lay.C);
  if (int rc = check_launch("seg_stats_kernel")) return rc;
  seg_keep_kernel<<<ids, kSegThreads, 0, st>>>(w, lay.C, T2, min_area, tau_hi);
  if (int rc = check_launch("seg_keep_kernel")) return rc;
  seg_scan_kernel<<<N, kSegScanThreads, 0, st>>>(w.ktiles, T2, w.tot, 1, w.acc, max_objects, count, dropped);
  if (int rc = check_launch("seg_scan_kernel")) return rc;
  seg_assign_kernel<<<ids, kSegThreads, 0, st>>>(w, lay.C, T2, min_area, tau_hi, max_objects);
  if (int rc = check_launch("seg_assign_kernel")) return rc;
  seg_label_kernel<<<tiles, kSegThreads, 0, st>>>(res_a, occ_a, reinterpret_cast<const float2*>(flow_a), affine_a, w,
                                                  labels, W, HW, lay.C, S);
  if (int rc = check_launch("seg_label_kernel")) return rc;
  seg_objects_kernel<<<N, kSegThreads, 0, st>>>(w.acc, count, objects, max_objects, S);
  return check_launch("seg_objects_kernel");
}
#endif  // !MFN_HOST_EMULATION
