// interp.cu -- frame interpolation from bidirectional flow: occlusion-weighted forward (average) splatting.
//
//   mfn_interpolate_frames   img0, img1 (N,H,W,3) uint8, flow_fw, flow_bw (N,H,W,2) (x,y) pixels, occ_fw, occ_bw (N,H,W)
//                            uint8, T host times in (0,1)  ->  out (N,T,H,W,3) uint8
//     per time step, over one step's workspace of int64 accumulators (N,H,W,4) (3 colour sums and the weight sum):
//       cudaMemsetAsync;  splat_kernel, grid (pixels / 256, N, 2), blockIdx.z picks the source image: each source pixel
//       adds its weighted colour to the (up to) four pixels around its target with integer atomics;  normalise_kernel,
//       grid (pixels / 256, N): one thread per output pixel writes out[:, k].
//     The rule is in include/maskflow_b200.h.  The sums are 64-bit fixed point (det.cuh), so they do not depend on the order
//     in which the atomics land: the output is bit-reproducible, and t travels by value, so the sequence is capture-safe.
//
// Scales (static: no max pass).  A destination receives at most one contribution per source pixel, so its fan-in is below
// 2^k with k = det_bits(2 H W).  Weights b w <= 1 use s_w = 61 - k; colours b w I <= 255 < 2^8 use s_c = s_w - 8.  Then every
// scaled contribution is below 2^(61-k) and no sum reaches 2^62.
//
// The file also builds for the host (MFN_HOST_EMULATION: tests/host_emu/interp_emu.cpp), one thread at a time.
#ifdef MFN_HOST_EMULATION
#include "cuda_shim.h"
#include "det.cuh"
#include "sampling.cuh"
#else
#include <math.h>

#include "common.cuh"
#include "det.cuh"
#endif

namespace mfn {

constexpr int kInterpHoleShift = 20;   // a pixel whose weight sum is below 2^-20 is a hole

// s_w of an H x W frame pair (s_c = s_w - 8)
static inline int interp_weight_shift(int H, int W) { return 61 - det_bits(2LL * H * W); }

// grid (ceil(HW / blockDim), N, 2): z = 0 splats img0's pixels along t * flow_fw with weight (1 - t), z = 1 img1's along
// (1 - t) * flow_bw with weight t; occluded sources are weighted by occ_weight.  acc (N,H,W,4): r, g, b, weight.
__global__ void __launch_bounds__(256)
    splat_kernel(const unsigned char* __restrict__ img0, const unsigned char* __restrict__ img1,
                 const float2* __restrict__ flow_fw, const float2* __restrict__ flow_bw,
                 const unsigned char* __restrict__ occ_fw, const unsigned char* __restrict__ occ_bw,
                 unsigned long long* __restrict__ acc, int H, int W, float t, float occ_weight, int s_w) {
  const int HW = H * W;
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= HW) return;
  const bool back = blockIdx.z != 0;
  const size_t n = blockIdx.y;
  const size_t i = n * HW + p;
  const float omt = 1.f - t;
  const float2 uv = __ldg((back ? flow_bw : flow_fw) + i);
  const float tt = back ? omt : t;
  const int y = p / W, x = p - y * W;
  const float qx = fmaf(tt, uv.x, (float)x), qy = fmaf(tt, uv.y, (float)y);
  // non-finite or beyond the one-pixel margin: no corner inside (checked before any float -> int conversion)
  if (!(qx >= -1.f && qx <= (float)W && qy >= -1.f && qy <= (float)H)) return;
  const float w = (back ? t : omt) * (__ldg((back ? occ_bw : occ_fw) + i) ? occ_weight : 1.f);
  const unsigned char* px = (back ? img1 : img0) + 3 * i;
  const float c0 = (float)__ldg(px), c1 = (float)__ldg(px + 1), c2 = (float)__ldg(px + 2);
  int off[4];
  float b[4];
  sampler_taps(qx, qy, H, W, off, b);   // a corner outside the frame has weight 0
  const FixedScale fw = det_fixed_scale(s_w), fc = det_fixed_scale(s_w - 8);
  unsigned long long* a = acc + 4 * n * HW;
  for (int k = 0; k < 4; ++k) {
    if (b[k] == 0.f) continue;          // outside the frame (dropped), or a corner the target lies a full pixel from
    const float bw = b[k] * w;
    unsigned long long* d = a + 4 * (size_t)off[k];
    atomicAdd(d + 0, det_to_fixed(bw * c0, fc));
    atomicAdd(d + 1, det_to_fixed(bw * c1, fc));
    atomicAdd(d + 2, det_to_fixed(bw * c2, fc));
    atomicAdd(d + 3, det_to_fixed(bw, fw));
  }
}

// grid (ceil(HW / blockDim), N): out (N,T,H,W,3) slice k.  Weight sum >= 2^-20: rint(colour / weight) (one double rounding,
// one float rounding, ties to even), clamped to [0,255]; below: the hole takes rint((1 - t) img0 + t img1).
__global__ void __launch_bounds__(256)
    normalise_kernel(const unsigned long long* __restrict__ acc, const unsigned char* __restrict__ img0,
                     const unsigned char* __restrict__ img1, unsigned char* __restrict__ out, int H, int W, int T, int k,
                     float t, int s_w) {
  const int HW = H * W;
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= HW) return;
  const size_t n = blockIdx.y;
  const size_t i = n * HW + p;
  const ulonglong2* a2 = reinterpret_cast<const ulonglong2*>(acc) + 2 * i;
  const ulonglong2 rg = __ldg(a2), bw = __ldg(a2 + 1);
  const long long cw = (long long)bw.y;
  unsigned char* o = out + 3 * ((n * T + k) * (size_t)HW + p);
  if (cw < (1LL << (s_w - kInterpHoleShift))) {
    const float omt = 1.f - t;
    const unsigned char* p0 = img0 + 3 * i;
    const unsigned char* p1 = img1 + 3 * i;
    for (int c = 0; c < 3; ++c) o[c] = (unsigned char)rintf(fmaf(t, (float)__ldg(p1 + c), omt * (float)__ldg(p0 + c)));
    return;
  }
  const long long cc[3] = {(long long)rg.x, (long long)rg.y, (long long)bw.x};
  for (int c = 0; c < 3; ++c) {
    const float v = rintf((float)((double)cc[c] / (double)cw * 256.0));   // 256 = 2^(s_w - s_c): exact
    o[c] = (unsigned char)fminf(fmaxf(v, 0.f), 255.f);
  }
}

}  // namespace mfn

#ifndef MFN_HOST_EMULATION
extern "C" long long mfn_interpolate_frames_workspace_bytes(int N, int H, int W) {
  return (N > 0 && H > 0 && W > 0) ? 32LL * N * H * W : 0;
}

extern "C" int mfn_interpolate_frames(const unsigned char* img0, const unsigned char* img1, const float* flow_fw,
                                      const float* flow_bw, const unsigned char* occ_fw, const unsigned char* occ_bw,
                                      unsigned char* out, void* ws, long long ws_bytes, int N, int H, int W,
                                      const float* times_host, int T, float occ_weight, void* stream) {
  using namespace mfn;
  MFN_REQUIRE(img0 && img1 && flow_fw && flow_bw && occ_fw && occ_bw && out && ws && times_host, MFN_ERR_INVALID_ARG,
              "mfn_interpolate_frames: null pointer");
  MFN_REQUIRE(N > 0 && H > 0 && W > 0, MFN_ERR_INVALID_ARG, "mfn_interpolate_frames: non-positive extent");
  MFN_REQUIRE(T > 0, MFN_ERR_INVALID_ARG, "mfn_interpolate_frames: T must be >= 1");
  for (int k = 0; k < T; ++k)
    MFN_REQUIRE(times_host[k] > 0.f && times_host[k] < 1.f, MFN_ERR_INVALID_ARG,
                "mfn_interpolate_frames: time %d is %g, outside (0,1)", k, (double)times_host[k]);
  MFN_REQUIRE(occ_weight >= 0.f && occ_weight <= 1.f, MFN_ERR_INVALID_ARG,
              "mfn_interpolate_frames: occ_weight must lie in [0,1], got %g", (double)occ_weight);
  MFN_REQUIRE(aligned(flow_fw, 8) && aligned(flow_bw, 8) && aligned(ws, 16), MFN_ERR_INVALID_ARG,
              "mfn_interpolate_frames: flow_fw and flow_bw must be 8-byte aligned, ws 16-byte aligned");
  MFN_REQUIRE((long long)H * W < (1LL << 31) && N <= 65535, MFN_ERR_ALIGNMENT,
              "mfn_interpolate_frames: extents overflow kernel indexing");
  const long long need = mfn_interpolate_frames_workspace_bytes(N, H, W);
  MFN_REQUIRE(ws_bytes >= need, MFN_ERR_INVALID_ARG, "mfn_interpolate_frames: workspace of %lld bytes, %lld needed",
              ws_bytes, need);
  const int HW = H * W;
  const int s_w = interp_weight_shift(H, W);
  cudaStream_t st = as_stream(stream);
  auto* acc = static_cast<unsigned long long*>(ws);
  for (int k = 0; k < T; ++k) {
    const float t = times_host[k];
    const cudaError_t ce = cudaMemsetAsync(ws, 0, (size_t)need, st);
    if (ce != cudaSuccess) return fail((int)ce, "mfn_interpolate_frames: cudaMemsetAsync: %s", cudaGetErrorString(ce));
    splat_kernel<<<dim3((HW + 255) / 256, N, 2), 256, 0, st>>>(
        img0, img1, reinterpret_cast<const float2*>(flow_fw), reinterpret_cast<const float2*>(flow_bw), occ_fw, occ_bw,
        acc, H, W, t, occ_weight, s_w);
    if (int rc = check_launch("splat_kernel")) return rc;
    normalise_kernel<<<dim3((HW + 255) / 256, N), 256, 0, st>>>(acc, img0, img1, out, H, W, T, k, t, s_w);
    if (int rc = check_launch("normalise_kernel")) return rc;
  }
  return 0;
}
#endif  // !MFN_HOST_EMULATION
