// unsup_loss_emu.cpp -- TEST INFRASTRUCTURE ONLY.  Compiles the census and smoothness loss kernels
// (maskflownet_b200/csrc/unsup_loss.cu) for the host through cuda_shim.h and runs them over the grids of their entry
// points, one thread per block (each thread's loop then covers the whole tile, and the tree reductions are serial);
// C ABI for tests/test_unsup_loss.py.
//   g++ -O1 -ffp-contract=off -shared -fPIC -I tests/host_emu unsup_loss_emu.cpp
#define MFN_HOST_EMULATION 1

#include "cuda_shim.h"
#include "../../maskflownet_b200/csrc/unsup_loss.cu"

#include <vector>

using namespace mfn::unsup;

#define EMU_API extern "C" __attribute__((visibility("default")))

static void finish(const float* partial, int parts, float* loss, float* vsum, int N, int H, int W) {
  gridDim = dim3(N);
  blockDim = dim3(1);
  threadIdx = dim3(0);
  for (int n = 0; n < N; ++n) {
    blockIdx = dim3(n);
    finish_kernel(partial, parts, loss, vsum, H, W);
  }
}

EMU_API void emu_census_forward(const float* img1, const float* img2w, const unsigned char* occ, float* coef, float* vsum,
                                float* loss, int N, int H, int W) {
  gridDim = dim3((W + TW - 1) / TW, (H + TH - 1) / TH, N);
  blockDim = dim3(1);
  threadIdx = dim3(0);
  const int parts = gridDim.x * gridDim.y;
  std::vector<float> partial((size_t)2 * N * parts);
  for (unsigned n = 0; n < gridDim.z; ++n)
    for (unsigned by = 0; by < gridDim.y; ++by)
      for (unsigned bx = 0; bx < gridDim.x; ++bx) {
        blockIdx = dim3(bx, by, n);
        census_forward_kernel(img1, img2w, occ, coef, partial.data(), H, W);
      }
  finish(partial.data(), parts, loss, vsum, N, H, W);
}

// d(p) at the interior pixels (0 elsewhere): the kernel's census_distance on whole grey planes made by its grey()
EMU_API void emu_census_distance(const float* img1, const float* img2w, float* d, int N, int H, int W) {
  const size_t plane = (size_t)H * W;
  std::vector<float> g1(plane), g2(plane);
  for (int n = 0; n < N; ++n) {
    for (size_t i = 0; i < plane; ++i) {
      g1[i] = grey(img1 + (size_t)n * 3 * plane, plane, i);
      g2[i] = grey(img2w + (size_t)n * 3 * plane, plane, i);
    }
    for (int y = 0; y < H; ++y)
      for (int x = 0; x < W; ++x) {
        const size_t i = (size_t)y * W + x;
        d[n * plane + i] = census_interior(x, y, H, W) ? census_distance(g1.data() + i, g2.data() + i, W) : 0.f;
      }
  }
}

EMU_API void emu_census_backward(const float* img1, const float* img2w, const float* coef, const float* vsum,
                                 const float* g_loss, float* g_img2w, int N, int H, int W) {
  gridDim = dim3((W + TW - 1) / TW, (H + TH - 1) / TH, N);
  blockDim = dim3(1);
  threadIdx = dim3(0);
  for (unsigned n = 0; n < gridDim.z; ++n)
    for (unsigned by = 0; by < gridDim.y; ++by)
      for (unsigned bx = 0; bx < gridDim.x; ++bx) {
        blockIdx = dim3(bx, by, n);
        census_backward_kernel(img1, img2w, coef, vsum, g_loss, g_img2w, H, W);
      }
}

EMU_API void emu_smoothness_forward(const float* flow, const float* img, float* loss, int N, int H, int W) {
  const int parts = (int)(((long long)H * W + SNT - 1) / SNT);
  std::vector<float> partial((size_t)2 * N * parts);
  gridDim = dim3(parts, N);
  blockDim = dim3(1);
  threadIdx = dim3(0);
  for (int n = 0; n < N; ++n)
    for (int b = 0; b < parts; ++b) {
      blockIdx = dim3(b, n);
      smoothness_forward_kernel(flow, img, partial.data(), H, W);
    }
  finish(partial.data(), parts, loss, nullptr, N, H, W);
}

EMU_API void emu_smoothness_backward(const float* flow, const float* img, const float* g_loss, float* g_flow, int N, int H,
                                     int W) {
  const int parts = (int)(((long long)H * W + SNT - 1) / SNT);
  gridDim = dim3(parts, N);
  blockDim = dim3(1);
  threadIdx = dim3(0);
  for (int n = 0; n < N; ++n)
    for (int b = 0; b < parts; ++b) {
      blockIdx = dim3(b, n);
      smoothness_backward_kernel(flow, img, g_loss, g_flow, H, W);
    }
}
