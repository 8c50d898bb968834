// consistency_emu.cpp -- TEST INFRASTRUCTURE ONLY.  Compiles the forward-backward consistency check
// (maskflownet_b200/csrc/consistency.cu) for the host through cuda_shim.h and runs it thread by thread over the grid of
// mfn_flow_consistency; C ABI for tests/test_bidirectional.py.
//   g++ -O1 -ffp-contract=off -shared -fPIC -I tests/host_emu consistency_emu.cpp
#define MFN_HOST_EMULATION 1

#include "cuda_shim.h"

// the vector type the kernel reads; floorf is the C library's
struct float2 {
  float x, y;
};

#include "../../maskflownet_b200/csrc/consistency.cu"

using namespace mfn;

#define EMU_API extern "C" __attribute__((visibility("default")))

EMU_API void emu_flow_consistency(const float* flow_fw, const float* flow_bw, unsigned char* occ_fw,
                                  unsigned char* occ_bw, int N, int H, int W, float alpha, float beta) {
  const int HW = H * W;
  blockDim = dim3(256);
  gridDim = dim3((HW + 255) / 256, N, 2);
  for (unsigned z = 0; z < gridDim.z; ++z)
    for (unsigned n = 0; n < gridDim.y; ++n)
      for (unsigned b = 0; b < gridDim.x; ++b) {
        blockIdx = dim3(b, n, z);
        for (unsigned t = 0; t < blockDim.x; ++t) {
          threadIdx = dim3(t);
          flow_consistency_kernel(reinterpret_cast<const float2*>(flow_fw), reinterpret_cast<const float2*>(flow_bw),
                                  occ_fw, occ_bw, H, W, alpha, beta);
        }
      }
}
