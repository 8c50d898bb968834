// consistency.cu -- forward-backward consistency check of a pair of flows (Sundaram, Brox and Keutzer, ECCV 2010): the
// pixels of each image that have no consistent match in the other.
//
//   mfn_flow_consistency   flow_fw, flow_bw (N,H,W,2) (x,y) pixels  ->  occ_fw, occ_bw (N,H,W) uint8 {0,1}
//     one launch, grid (pixels / 256, N, 2): blockIdx.z picks the direction.  One thread per pixel: follow its own flow,
//     sample the other direction's flow bilinearly at the target, and compare the round trip with the flows' magnitude.
//     No atomics and no shared memory: every output byte is written once by one thread, so the result is deterministic.
//
// The file also builds for the host (MFN_HOST_EMULATION: tests/host_emu/consistency_emu.cpp), one thread at a time.
#ifdef MFN_HOST_EMULATION
#include "cuda_shim.h"
#else
#include <math.h>

#include "common.cuh"
#endif
#include "flowcheck.cuh"   // fb_occluded

namespace mfn {

// grid (ceil(HW / blockDim), N, 2): z = 0 writes occ_fw from flow_fw against flow_bw, z = 1 the reverse.
__global__ void __launch_bounds__(256)
    flow_consistency_kernel(const float2* __restrict__ flow_fw, const float2* __restrict__ flow_bw,
                            unsigned char* __restrict__ occ_fw, unsigned char* __restrict__ occ_bw, int H, int W,
                            float alpha, float beta) {
  const int HW = H * W;
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= HW) return;
  const bool back = blockIdx.z != 0;
  const size_t base = (size_t)blockIdx.y * HW;
  const float2* self = (back ? flow_bw : flow_fw) + base;
  const float2* other = (back ? flow_fw : flow_bw) + base;
  const int y = p / W, x = p - y * W;
  (back ? occ_bw : occ_fw)[base + p] = fb_occluded(other, H, W, x, y, __ldg(self + p), alpha, beta);
}

}  // namespace mfn

#ifndef MFN_HOST_EMULATION
extern "C" int mfn_flow_consistency(const float* flow_fw, const float* flow_bw, unsigned char* occ_fw,
                                    unsigned char* occ_bw, int N, int H, int W, float alpha, float beta, void* stream) {
  using namespace mfn;
  MFN_REQUIRE(flow_fw && flow_bw && occ_fw && occ_bw, MFN_ERR_INVALID_ARG, "mfn_flow_consistency: null pointer");
  MFN_REQUIRE(N > 0 && H > 0 && W > 0, MFN_ERR_INVALID_ARG, "mfn_flow_consistency: non-positive extent");
  MFN_REQUIRE(aligned(flow_fw, 8) && aligned(flow_bw, 8), MFN_ERR_INVALID_ARG,
              "mfn_flow_consistency: flow_fw and flow_bw must be 8-byte aligned");
  MFN_REQUIRE(isfinite(alpha) && alpha >= 0.f && isfinite(beta) && beta >= 0.f, MFN_ERR_INVALID_ARG,
              "mfn_flow_consistency: alpha and beta must be finite and non-negative");
  MFN_REQUIRE((long long)H * W < (1LL << 31) && N <= 65535, MFN_ERR_ALIGNMENT,
              "mfn_flow_consistency: extents overflow kernel indexing");
  const int HW = H * W;
  flow_consistency_kernel<<<dim3((HW + 255) / 256, N, 2), 256, 0, as_stream(stream)>>>(
      reinterpret_cast<const float2*>(flow_fw), reinterpret_cast<const float2*>(flow_bw), occ_fw, occ_bw, H, W, alpha,
      beta);
  return check_launch("flow_consistency_kernel");
}
#endif  // !MFN_HOST_EMULATION
