// flowvis.cu -- Middlebury colour coding of a flow field (Baker et al.; the flow_vis.flow_to_color convention that the
// reference's predict_new_data.py writes), so that a video of flows can be coloured on the GPU and leave it as uint8.
//
//   mfn_flow_to_color   flow (N,H,W,2) (x,y) pixels  ->  rgb (N,H,W,3) uint8, rad_max (N)
//     radius pass   (only without a fixed max_radius) per sample max of sqrt(u^2+v^2): grid-stride, warp max, one
//                   atomicMax per warp on the float's bit pattern (non-negative floats order like their bits; max is
//                   order-independent, so the result is deterministic)
//     colour pass   one thread per pixel: normalise, angle -> position on the 55-entry colour wheel, blend the two
//                   neighbouring entries, whiten towards the centre (radius <= 1) or darken outside it
//
// The file also builds for the host (MFN_HOST_EMULATION: tests/host_emu/flowvis_emu.cpp), one thread at a time.
#ifdef MFN_HOST_EMULATION
#include "cuda_shim.h"
#else
#include <math.h>

#include "common.cuh"
#endif

namespace mfn {

constexpr int kWheelSize = 55;

// segments RY 15, YG 6, GC 4, CB 11, BM 13, MR 6; entry i of a segment of length L ramps one channel by floor(255 i / L)
__constant__ unsigned char kFlowWheel[kWheelSize * 3] = {
    /* RY */ 255, 0, 0, 255, 17, 0, 255, 34, 0, 255, 51, 0, 255, 68, 0, 255, 85, 0, 255, 102, 0, 255, 119, 0, 255, 136, 0,
    255, 153, 0, 255, 170, 0, 255, 187, 0, 255, 204, 0, 255, 221, 0, 255, 238, 0,
    /* YG */ 255, 255, 0, 213, 255, 0, 170, 255, 0, 128, 255, 0, 85, 255, 0, 43, 255, 0,
    /* GC */ 0, 255, 0, 0, 255, 63, 0, 255, 127, 0, 255, 191,
    /* CB */ 0, 255, 255, 0, 232, 255, 0, 209, 255, 0, 186, 255, 0, 163, 255, 0, 140, 255, 0, 116, 255, 0, 93, 255, 0, 70, 255,
    0, 47, 255, 0, 24, 255,
    /* BM */ 0, 0, 255, 19, 0, 255, 39, 0, 255, 58, 0, 255, 78, 0, 255, 98, 0, 255, 117, 0, 255, 137, 0, 255, 156, 0, 255,
    176, 0, 255, 196, 0, 255, 215, 0, 255, 235, 0, 255,
    /* MR */ 255, 0, 255, 255, 0, 213, 255, 0, 170, 255, 0, 128, 255, 0, 85, 255, 0, 43,
};

// u^2 + v^2 without contraction: both passes must compute it identically (see the colour kernel)
__device__ __forceinline__ float sq_radius(float2 uv) { return __fadd_rn(__fmul_rn(uv.x, uv.x), __fmul_rn(uv.y, uv.y)); }

// grid (bx, N): blocks of row n reduce sample n into rad_max[n], which must hold +0 on entry.  blockDim: a multiple of 32.
// NaN pixels are skipped (fmaxf returns the other operand).
__global__ void __launch_bounds__(256)
    flow_radius_max_kernel(const float2* __restrict__ flow, float* __restrict__ rad_max, int HW) {
  const int n = blockIdx.y;
  const float2* f = flow + (size_t)n * HW;
  float m = 0.f;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < HW; i += (long long)gridDim.x * blockDim.x)
    m = fmaxf(m, sq_radius(__ldg(f + i)));
  m = sqrtf(m);   // sqrt is monotone: the sqrt of the max is the max of the radii
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) atomicMax(reinterpret_cast<unsigned*>(rad_max + n), __float_as_uint(m));
}

// Position of a normalised (u, v) on the wheel: blend of entries k0 and k1 with weight f on k1.  fmaxf / fminf return
// the non-NaN operand, and k0 is clamped too: every input, NaN and inf included, indexes inside the table.
__device__ __forceinline__ void wheel_taps(float u, float v, int& k0, int& k1, float& f) {
  const float a = atan2f(-v, -u) / 3.14159265358979f;   // literal negations: the sign of a zero picks entry 0 or 54
  const float fk = fminf(fmaxf((a + 1.f) / 2.f * (float)(kWheelSize - 1), 0.f), (float)(kWheelSize - 1));
  k0 = min(max((int)floorf(fk), 0), kWheelSize - 1);
  k1 = k0 + 1 == kWheelSize ? 0 : k0 + 1;
  f = fk - (float)k0;
}

// One thread per pixel.  max_radius > 0: fixed scale, written to rad_max; else rad_max holds the measured radius.
__global__ void __launch_bounds__(256)
    flow_to_color_kernel(const float2* __restrict__ flow, unsigned char* __restrict__ rgb, float* __restrict__ rad_max,
                         int HW, unsigned total, float max_radius, int bgr) {
  // the wheel staged in shared memory, one packed R | G << 8 | B << 16 word per entry: lanes of a warp read different
  // entries wherever the flow's direction varies between neighbours, which constant memory would serialise
  __shared__ unsigned wheel[kWheelSize];
  for (int i = threadIdx.x; i < kWheelSize; i += blockDim.x)
    wheel[i] = kFlowWheel[3 * i] | (unsigned)kFlowWheel[3 * i + 1] << 8 | (unsigned)kFlowWheel[3 * i + 2] << 16;
  __syncthreads();
  const unsigned idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int n = (int)(idx / (unsigned)HW);
  const bool fixed = max_radius > 0.f;
  if (fixed && idx - (unsigned)n * HW == 0) rad_max[n] = max_radius;
  const float2 uv = __ldg(flow + idx);
  const float d = fixed ? max_radius : __ldg(rad_max + n) + 1e-5f;
  const float u = uv.x / d, v = uv.y / d;
  // the radius of the normalised flow, taken as sqrt(u^2+v^2) / d rather than from the rounded quotients: sqrt(u^2+v^2)
  // is at most the measured maximum r <= r + 1e-5, so no pixel of a per-sample normalisation lands outside the unit disc
  const float rad = sqrtf(sq_radius(uv)) / d;
  int k0, k1;
  float f;
  wheel_taps(u, v, k0, k1, f);
  const unsigned w0 = wheel[k0], w1 = wheel[k1];
  unsigned char* out = rgb + (size_t)idx * 3;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    float col = ((1.f - f) * (float)((w0 >> 8 * c) & 255u) + f * (float)((w1 >> 8 * c) & 255u)) / 255.f;
    col = rad <= 1.f ? 1.f - rad * (1.f - col) : col * 0.75f;
    out[bgr ? 2 - c : c] = (unsigned char)fminf(fmaxf(floorf(255.f * col), 0.f), 255.f);
  }
}

}  // namespace mfn

#ifndef MFN_HOST_EMULATION
extern "C" int mfn_flow_to_color(const float* flow_xy, unsigned char* rgb, float* rad_max, int N, int H, int W,
                                 float max_radius, int bgr, void* stream) {
  using namespace mfn;
  MFN_REQUIRE(flow_xy && rgb && rad_max, MFN_ERR_INVALID_ARG, "mfn_flow_to_color: null pointer");
  MFN_REQUIRE(N > 0 && H > 0 && W > 0, MFN_ERR_INVALID_ARG, "mfn_flow_to_color: non-positive extent");
  MFN_REQUIRE(isfinite(max_radius), MFN_ERR_INVALID_ARG, "mfn_flow_to_color: max_radius must be finite");
  MFN_REQUIRE((long long)N * H * W < (1LL << 31) && N <= 65535, MFN_ERR_ALIGNMENT,
              "mfn_flow_to_color: extents overflow kernel indexing");
  MFN_REQUIRE(aligned(flow_xy, 8), MFN_ERR_ALIGNMENT, "mfn_flow_to_color: flow_xy must be 8-byte aligned");
  cudaStream_t st = as_stream(stream);
  const int HW = H * W;
  const float2* flow = reinterpret_cast<const float2*>(flow_xy);
  if (!(max_radius > 0.f)) {
    const cudaError_t ce = cudaMemsetAsync(rad_max, 0, sizeof(float) * N, st);
    if (ce != cudaSuccess) return fail((int)ce, "mfn_flow_to_color: cudaMemsetAsync: %s", cudaGetErrorString(ce));
    // one wave of 256-thread blocks across the samples
    const int per_sample = (kNumSMs * 8 + N - 1) / N;
    const int bx = (HW + 255) / 256 < per_sample ? (HW + 255) / 256 : per_sample;
    flow_radius_max_kernel<<<dim3(bx, N), 256, 0, st>>>(flow, rad_max, HW);
    const int rc = check_launch("flow_radius_max_kernel");
    if (rc) return rc;
  }
  const unsigned total = (unsigned)N * (unsigned)HW;
  flow_to_color_kernel<<<(total + 255) / 256, 256, 0, st>>>(flow, rgb, rad_max, HW, total, max_radius, bgr ? 1 : 0);
  return check_launch("flow_to_color_kernel");
}
#endif  // !MFN_HOST_EMULATION
