// stabilize_emu.cpp -- TEST INFRASTRUCTURE ONLY.  Compiles video stabilisation (maskflownet_b200/csrc/stabilize.cu) for the
// host through cuda_shim.h and runs the launch sequences of mfn_affine_motion and mfn_warp_frames_affine one thread at a
// time.  The reduction kernels' phases run over their 256 threads in turn, with the same tree steps in between;
// C ABI for tests/test_stabilize.py.
//   g++ -O1 -ffp-contract=off -shared -fPIC -I tests/host_emu stabilize_emu.cpp
#define MFN_HOST_EMULATION 1
#include <cstring>
#include <vector>

#include "cuda_shim.h"

// the vector type and the bit cast the kernels use; floor, rint, sqrt, fmin and fmax are the C library's
struct float2 {
  float x, y;
};
static inline float __int_as_float(int v) {
  float f;
  std::memcpy(&f, &v, 4);
  return f;
}

#include "../../maskflownet_b200/csrc/stabilize.cu"

using namespace mfn;

#define EMU_API extern "C" __attribute__((visibility("default")))

EMU_API int emu_fit_ctas(int H, int W) { return fit_ctas(H, W); }

// mfn_affine_motion's launches: per iteration the accumulation over G CTAs per sample and the solve, then the residual
EMU_API void emu_affine_motion(const float* flow, double* affine, unsigned char* ok, float* residual, int N, int H, int W,
                               int iterations, float sigma) {
  const int T = kFitThreads, G = fit_ctas(H, W), HW = H * W;
  const float2* f2 = reinterpret_cast<const float2*>(flow);
  std::vector<double> part((size_t)N * G * kFitMoments);
  static double sh[kFitThreads][kFitMoments];
  for (int k = 0; k < iterations; ++k) {
    const double sk = (double)sigma * (double)(1 << (k < 4 ? 4 - k : 0));
    const double inv_sig2 = k == 0 ? 0.0 : 1.0 / (sk * sk);
    for (int n = 0; n < N; ++n)
      for (int g = 0; g < G; ++g) {
        for (int t = 0; t < T; ++t) fit_thread_sums(f2 + (size_t)n * HW, affine + 6 * n, H, W, g, G, t, inv_sig2, sh[t]);
        for (int stride = T / 2; stride > 0; stride >>= 1)
          for (int t = 0; t < T; ++t) fit_tree_step(sh, t, stride);
        std::memcpy(&part[((size_t)n * G + g) * kFitMoments], sh[0], sizeof(sh[0]));
      }
    for (int n = 0; n < N; ++n) {
      for (int t = 0; t < T; ++t) fit_partial_sums(&part[(size_t)n * G * kFitMoments], G, t, sh[t]);
      for (int stride = T / 2; stride > 0; stride >>= 1)
        for (int t = 0; t < T; ++t) fit_tree_step(sh, t, stride);
      fit_solve(sh[0], H, W, affine + 6 * n, ok + n);
    }
  }
  if (!residual) return;
  blockDim = dim3(256);
  gridDim = dim3((HW + 255) / 256, N);
  for (unsigned n = 0; n < (unsigned)N; ++n)
    for (unsigned b = 0; b < gridDim.x; ++b)
      for (unsigned t = 0; t < 256; ++t) {
        blockIdx = dim3(b, n);
        threadIdx = dim3(t);
        fit_residual_kernel(f2, affine, residual, H, W);
      }
}

EMU_API void emu_warp_frames_affine(const unsigned char* src, const double* M, unsigned char* out, int N, int H, int W) {
  const int HW = H * W;
  blockDim = dim3(256);
  gridDim = dim3((HW + 255) / 256, N);
  for (unsigned n = 0; n < (unsigned)N; ++n)
    for (unsigned b = 0; b < gridDim.x; ++b)
      for (unsigned t = 0; t < 256; ++t) {
        blockIdx = dim3(b, n);
        threadIdx = dim3(t);
        warp_affine_kernel(src, M, out, H, W);
      }
}
