// flowvis_emu.cpp -- TEST INFRASTRUCTURE ONLY.  Compiles the flow colour coding (maskflownet_b200/csrc/flowvis.cu) for the
// host through cuda_shim.h and runs it thread by thread, in the launch order of mfn_flow_to_color; C ABI for
// tests/test_flow_visualization.py.
//   g++ -O1 -ffp-contract=off -shared -fPIC -I tests/host_emu flowvis_emu.cpp
#define MFN_HOST_EMULATION 1
#include <cstring>

#include "cuda_shim.h"

// what these kernels use beyond the shim: the vector type, the constant-memory qualifier, the bit cast, and the atomic,
// which with one thread at a time is a compare-and-store.  atan2f is the C library's.
#define __constant__
struct float2 {
  float x, y;
};
static inline unsigned __float_as_uint(float f) {
  unsigned u;
  std::memcpy(&u, &f, sizeof u);
  return u;
}
static inline unsigned atomicMax(unsigned* p, unsigned v) {
  const unsigned old = *p;
  if (v > old) *p = v;
  return old;
}

#include "../../maskflownet_b200/csrc/flowvis.cu"

using namespace mfn;

#define EMU_API extern "C" __attribute__((visibility("default")))

EMU_API void emu_wheel_taps(float u, float v, int* k0, int* k1, float* f) { wheel_taps(u, v, *k0, *k1, *f); }

EMU_API void emu_flow_to_color(const float* flow_xy, unsigned char* rgb, float* rad_max, int N, int H, int W,
                               float max_radius, int bgr) {
  const int HW = H * W;
  const float2* flow = reinterpret_cast<const float2*>(flow_xy);
  // one-thread blocks: the warp shuffle of the shim returns the thread's own value and every thread is a lane 0 (max
  // pass), and each block stages the whole shared-memory wheel before its barrier (colour pass)
  blockDim = dim3(1);
  threadIdx = dim3(0);
  if (!(max_radius > 0.f)) {
    std::memset(rad_max, 0, sizeof(float) * N);
    gridDim = dim3(5, N);
    for (int n = 0; n < N; ++n)
      for (unsigned b = 0; b < gridDim.x; ++b) {
        blockIdx = dim3(b, n);
        flow_radius_max_kernel(flow, rad_max, HW);
      }
  }
  const unsigned total = (unsigned)N * HW;
  gridDim = dim3(total);
  for (unsigned b = 0; b < gridDim.x; ++b) {
    blockIdx = dim3(b);
    flow_to_color_kernel(flow, rgb, rad_max, HW, total, max_radius, bgr);
  }
}
