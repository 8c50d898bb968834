// det_emu.cpp -- TEST INFRASTRUCTURE ONLY.  Compiles the deterministic backward mode -- the fixed-point arithmetic
// (maskflownet_b200/csrc/det.cuh), its shared passes (det_bwd.cu) and the deterministic BilinearSampler backward
// (image_warp_bwd.cu) -- for the host through cuda_shim.h, and runs the kernels one thread at a time in a caller-chosen
// order of threads; C ABI for tests/test_deterministic.py.
//   g++ -O1 -ffp-contract=off -shared -fPIC -I tests/host_emu det_emu.cpp
#define MFN_HOST_EMULATION 1
#include <vector>

#include "cuda_shim.h"

// what these kernels use beyond the shim and det.cuh's stand-ins: the fast exponential is the C library's (glibc declares an
// internal __expf of its own, hence the macro); with one thread at a time the atomics are plain read-modify-writes and the
// warp reduction returns the thread's own value
#define __expf expf
static inline float atomicAdd(float* p, float v) {
  const float old = *p;
  *p = old + v;
  return old;
}
static inline unsigned atomicMax(unsigned* p, unsigned v) {
  const unsigned old = *p;
  if (v > old) *p = v;
  return old;
}
static inline unsigned __reduce_max_sync(unsigned, unsigned v) { return v; }

#include "../../maskflownet_b200/csrc/det_bwd.cu"
#include "../../maskflownet_b200/csrc/image_warp_bwd.cu"

using namespace mfn;

#define EMU_API extern "C" __attribute__((visibility("default")))

// one-thread blocks, visited in the order `order` (a permutation of 0..nblocks-1; null = ascending)
template <typename F>
static void run_blocks(long long nblocks, const long long* order, F&& body) {
  gridDim = dim3((unsigned)nblocks);
  blockDim = dim3(1);
  threadIdx = dim3(0);
  for (long long i = 0; i < nblocks; ++i) {
    blockIdx = dim3((unsigned)(order ? order[i] : i));
    body();
  }
}

EMU_API int emu_det_bits(long long n) { return det_bits(n); }

// the scale det_scale derives from bound words b0 (and b1 when nb == 2): returns s (2^s = up), finite flag through *finite
EMU_API int emu_det_scale(float b0, float b1, int nb, int fanin_bits, int* finite) {
  const unsigned bound[2] = {det_abs_bits(b0), det_abs_bits(b1)};
  const FixedScale f = det_scale(bound, nb, fanin_bits);
  *finite = f.finite ? 1 : 0;
  int e = 0;
  frexpf(f.up, &e);
  return e - 1;
}

// mfn_bilinear_sampler_backward_det's launch sequence (zeroed workspace, max pass, scatter, conversion); the scatter's
// threads (one per output pixel) run in the order `order`.  grad_data is accumulated into, like the device entry point.
EMU_API void emu_bilinear_sampler_backward_det(const float* grad_out, const float* data, const float* grid, float* grad_data,
                                               float* grad_grid, int N, int C, int H, int W, int OH, int OW,
                                               const long long* order) {
  unsigned bound[2] = {0u, 0u};
  const long long n_acc = (long long)N * C * H * W, n_go = (long long)N * C * OH * OW, pix = (long long)N * OH * OW;
  std::vector<unsigned long long> acc(n_acc, 0ull);
  const int fanin_bits = det_bits(4LL * OH * OW);
  run_blocks(7, nullptr, [&] { det_abs_max_kernel(grad_out, n_go, bound); });
  run_blocks(pix, order, [&] {
    bilinear_sampler_bwd_det_kernel(grad_out, data, grid, grad_grid, N, C, H, W, OH, OW, acc.data(), bound, fanin_bits);
  });
  run_blocks(5, nullptr, [&] { det_fixed_to_float_kernel(acc.data(), grad_data, n_acc, bound, 1, fanin_bits); });
}

// the K4 bound: max over pixels of sum_f |g[n,f,pixel]|
EMU_API float emu_pixel_abs_sum_max(const float* g, int N, int F, long long HW) {
  unsigned bound = 0u;
  run_blocks(3, nullptr, [&] { det_pixel_abs_sum_max_kernel(g, N, F, HW, &bound); });
  return __uint_as_float(bound);
}

// det_ordered_sum_kernel with its threads (one per element) in the order `order`
EMU_API void emu_ordered_sum(const float* part, int nparts, long long part_stride, long long elem_stride, float* out,
                             long long n, int accumulate, const long long* order) {
  run_blocks(n, order, [&] { det_ordered_sum_kernel(part, nparts, part_stride, elem_stride, out, n, accumulate); });
}
