// image_warp_bwd_emu.cpp -- TEST INFRASTRUCTURE ONLY.  Compiles the image-warp backward kernels
// (maskflownet_b200/csrc/image_warp_bwd.cu, with the shared sampling.cuh) for the host through cuda_shim.h and runs them
// thread by thread; C ABI for tests/test_image_warp_backward.py.
//   g++ -O1 -ffp-contract=off -shared -fPIC -I tests/host_emu image_warp_bwd_emu.cpp
#define MFN_HOST_EMULATION 1
#include "cuda_shim.h"

// the two device intrinsics these kernels use beyond the shim: the fast exponential is the C library's (glibc declares an
// internal __expf of its own, hence the macro), and with one thread at a time the atomic is a plain add
#define __expf expf
static inline float atomicAdd(float* p, float v) {
  const float old = *p;
  *p = old + v;
  return old;
}

#include "../../maskflownet_b200/csrc/image_warp_bwd.cu"

using namespace mfn;

// a small grid of a few threads per block: fewer threads than items, so the grid-stride loops are exercised
template <typename F>
static void run(F&& body) {
  gridDim = dim3(5);
  blockDim = dim3(3);
  for (unsigned b = 0; b < gridDim.x; ++b)
    for (unsigned t = 0; t < blockDim.x; ++t) {
      blockIdx = dim3(b);
      threadIdx = dim3(t);
      body();
    }
}

#define EMU_API extern "C" __attribute__((visibility("default")))

EMU_API void emu_grid_generator_warp_backward(const float* grad_grid, float* grad_flow, int N, int H, int W) {
  run([&] { gridgen_warp_bwd_kernel(grad_grid, grad_flow, N, H, W); });
}

EMU_API void emu_bilinear_sampler_backward(const float* grad_out, const float* data, const float* grid, float* grad_data,
                                           float* grad_grid, int N, int C, int H, int W, int OH, int OW) {
  run([&] { bilinear_sampler_bwd_kernel(grad_out, data, grid, grad_data, grad_grid, N, C, H, W, OH, OW); });
}

EMU_API void emu_image_warp_concat_backward(const float* grad_c40, const float* im2, const float* flow_q, const float* mask_q,
                                            float* grad_im2, float* grad_flow_up, float* grad_mask_up, int N, int Ci, int H,
                                            int W, float flow_scale) {
  run([&] {
    image_warp_concat_bwd_kernel(grad_c40, im2, flow_q, mask_q, grad_im2, grad_flow_up, grad_mask_up, N, Ci, H, W,
                                 flow_scale);
  });
}
