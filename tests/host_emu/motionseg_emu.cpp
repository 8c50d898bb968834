// motionseg_emu.cpp -- TEST INFRASTRUCTURE ONLY.  Compiles moving-object segmentation (maskflownet_b200/csrc/motionseg.cu)
// for the host through cuda_shim.h and runs the launch sequence of mfn_motion_segment one thread at a time.  The tile
// kernels' phases run over their 256 threads in turn, with the block scans and reductions done here in between; the
// 1024-thread scan kernel is a serial scan here.  `seed` != 0 runs the per-pixel kernels (init, merge), the compression
// and the statistics in a shuffled order of pixels and threads, to show that the result does not depend on the order of
// the unions.  Every step of a find asserts parent[i] < i (motionseg.cu, SEG_ASSERT).
// C ABI for tests/test_motion_segment.py.
//   g++ -O1 -ffp-contract=off -shared -fPIC -I tests/host_emu motionseg_emu.cpp
#define MFN_HOST_EMULATION 1
#include <cstring>
#include <vector>

#include "cuda_shim.h"

// the vector type, bit casts, rounded double operations and integer atomics the kernels use
struct float2 {
  float x, y;
};
static inline float __int_as_float(int v) {
  float f;
  std::memcpy(&f, &v, 4);
  return f;
}
static inline unsigned __float_as_uint(float v) {
  unsigned u;
  std::memcpy(&u, &v, 4);
  return u;
}
static inline float __uint_as_float(unsigned v) {
  float f;
  std::memcpy(&f, &v, 4);
  return f;
}
static inline double __longlong_as_double(long long v) {
  double d;
  std::memcpy(&d, &v, 8);
  return d;
}
static inline double __dadd_rn(double a, double b) { volatile double r = a + b; return r; }
static inline double __dsub_rn(double a, double b) { volatile double r = a - b; return r; }
static inline double __dmul_rn(double a, double b) { volatile double r = a * b; return r; }
template <typename T>
static inline T atomicMin(T* p, T v) {
  const T old = *p;
  if (v < old) *p = v;
  return old;
}
template <typename T>
static inline T atomicMax(T* p, T v) {
  const T old = *p;
  if (v > old) *p = v;
  return old;
}
template <typename T>
static inline T atomicAdd(T* p, T v) {
  const T old = *p;
  *p = old + v;
  return old;
}
using std::isfinite;

#include "../../maskflownet_b200/csrc/motionseg.cu"

using namespace mfn;

#define EMU_API extern "C" __attribute__((visibility("default")))

// 0 .. n-1 in order (seed 0) or shuffled by a seeded linear congruential Fisher-Yates
static std::vector<int> order(int n, unsigned long long& seed) {
  std::vector<int> o(n);
  for (int i = 0; i < n; ++i) o[i] = i;
  if (seed == 0) return o;
  for (int i = n - 1; i > 0; --i) {
    seed = seed * 6364136223846793005ULL + 1442695040888963407ULL;
    const int j = (int)((seed >> 33) % (unsigned long long)(i + 1));
    const int t = o[i];
    o[i] = o[j];
    o[j] = t;
  }
  return o;
}

EMU_API long long emu_workspace_bytes(int N, int H, int W) { return seg_layout(N, H, W).bytes; }
EMU_API int emu_scale_bits(int H, int W) { return seg_scale_bits((long long)H * W); }

EMU_API void emu_motion_segment(const float* res_a, const unsigned char* occ_a, const float* res_b,
                                const unsigned char* occ_b, const float* flow_a, const double* affine_a,
                                unsigned char* labels, double* objects, int* count, int* dropped, int N, int H, int W,
                                float tau_lo, float tau_hi, int min_area, int max_objects, unsigned long long seed) {
  const SegLayout lay = seg_layout(N, H, W);
  const int HW = H * W, T1 = (int)lay.T1, T2 = (int)lay.T2, S = seg_scale_bits(lay.HW);
  const long long C = lay.C;
  std::vector<int> parent((size_t)N * HW), tiles((size_t)N * T1), ktiles((size_t)N * T2), tot(2 * (size_t)N);
  std::vector<unsigned> comp((size_t)N * C * 3);
  std::vector<SegAcc> acc((size_t)N * kSegMaxObjects);
  std::vector<int> part(kSegThreads);
  const float2* f2 = reinterpret_cast<const float2*>(flow_a);
  auto scan = [&](int* c, int T, int* total) {
    int run = 0;
    for (int i = 0; i < T; ++i) {
      const int v = c[i];
      c[i] = run;
      run += v;
    }
    *total = run;
  };
  // the exclusive scan of the 256 threads' counts of one tile
  auto block_scan = [&](const std::vector<int>& v, std::vector<int>& excl) {
    int run = 0;
    for (int t = 0; t < kSegThreads; ++t) excl[t] = run, run += v[t];
  };
  std::vector<int> excl(kSegThreads);
  for (int n = 0; n < N; ++n) {
    int* L = parent.data() + (size_t)n * HW;
    unsigned* cp = comp.data() + (size_t)n * C * 3;
    SegAcc* ac = acc.data() + (size_t)n * kSegMaxObjects;
    for (int p : order(HW, seed)) seg_init_pixel(res_a, occ_a, res_b, occ_b, parent.data(), HW, n, p, tau_lo);
    for (int p : order(HW, seed)) seg_merge_pixel(L, H, W, p);
    // seg_count_kernel: the tiles and their threads in any order, the tile's sum once all its threads ran
    for (int g : order(T1, seed)) {
      int total = 0;
      for (int t : order(kSegThreads, seed)) total += seg_compress_count(L, HW, g, t);
      tiles[(size_t)n * T1 + g] = total;
    }
    scan(&tiles[(size_t)n * T1], T1, &tot[2 * n]);
    for (int g = 0; g < T1; ++g) {
      for (int t = 0; t < kSegThreads; ++t) part[t] = seg_count_roots(L, HW, g, t);
      block_scan(part, excl);
      for (int t = 0; t < kSegThreads; ++t) seg_number_roots(L, cp, HW, g, t, tiles[(size_t)n * T1 + g] + excl[t]);
    }
    for (int g : order(T1, seed))
      for (int t : order(kSegThreads, seed)) seg_stats_run(res_a, occ_a, res_b, occ_b, L, cp, HW, n, g, t);
    const int R = tot[2 * n];
    for (int g = 0; g < T2; ++g) {
      int total = 0;
      for (int t = 0; t < kSegThreads; ++t) total += seg_count_kept(cp, R, g, t, min_area, tau_hi);
      ktiles[(size_t)n * T2 + g] = total;
    }
    scan(&ktiles[(size_t)n * T2], T2, &tot[2 * n + 1]);
    seg_clear_objects(ac, 0, 1, tot[2 * n + 1], max_objects, count + n, dropped + n);
    for (int g = 0; g < T2; ++g) {
      for (int t = 0; t < kSegThreads; ++t) part[t] = seg_count_kept(cp, R, g, t, min_area, tau_hi);
      block_scan(part, excl);
      for (int t = 0; t < kSegThreads; ++t)
        seg_assign(cp, ac, R, g, t, ktiles[(size_t)n * T2 + g] + excl[t], min_area, tau_hi, max_objects);
    }
    for (int g : order(T1, seed))
      for (int t : order(kSegThreads, seed))
        seg_label_run(res_a, occ_a, f2, affine_a, L, cp, ac, labels, W, HW, n, g, t, S);
    for (int j = 0; j < max_objects; ++j)
      seg_object_row(ac[j], j, count[n], S, objects + ((size_t)n * max_objects + j) * kSegObjCols);
  }
}

// The union-find alone on a foreground mask (N,H,W) uint8: the frame-local root of every pixel after the merge and the
// compression, -1 for the background.  The merge runs in the order of `seed`.
EMU_API void emu_union_find(const unsigned char* mask, int* roots, int N, int H, int W, unsigned long long seed) {
  const int HW = H * W;
  for (int n = 0; n < N; ++n) {
    int* L = roots + (size_t)n * HW;
    for (int p = 0; p < HW; ++p) L[p] = mask[(size_t)n * HW + p] ? p : -1;
    for (int p : order(HW, seed)) seg_merge_pixel(L, H, W, p);
    const int T1 = (HW + kSegTile - 1) / kSegTile;
    for (int g = 0; g < T1; ++g)
      for (int t = 0; t < kSegThreads; ++t) seg_compress_count(L, HW, g, t);
  }
}
