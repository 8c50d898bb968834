// det_bwd.cu -- the order-independent passes of the deterministic backward mode (maskflow_b200.h: the *_det entry points,
// arithmetic in det.cuh).  The entry points themselves live next to their atomic counterparts (warp_bwd.cu,
// image_warp_bwd.cu, prepost.cu), whose kernels take a DET template flag; this file holds what they share:
//
//   det_abs_max_kernel            bound[0] = max |v| over a tensor
//   det_pixel_abs_sum_max_kernel  bound[0] = max over pixels of sum_f |g[n,f,pixel]|  (the K4 bound: |g_S| <= that * max|W|)
//       grid-stride, a warp max of the bit patterns (det_abs_bits), one atomicMax per warp: max is order-independent, so the
//       bound is the same whatever the grid; NaN is kept (it orders above +inf).  bound must hold 0 on entry.
//   det_fixed_to_float_kernel     out[i] += the fp32 value of the int64 fixed-point sum acc[i] (NaN for a non-finite scale)
//   det_ordered_sum_kernel        out[e] (+)= sum_{b = 0 .. nparts-1} part[e * elem_stride + b * part_stride], one thread per
//       element walking the parts in index order: the order is fixed by the partition, which the callers derive from the
//       shape alone (never from the SM count), so the result does not depend on the GPU or the grid.
//
// The file also builds for the host (MFN_HOST_EMULATION: tests/host_emu/det_emu.cpp), one thread at a time.
#ifdef MFN_HOST_EMULATION
#include "cuda_shim.h"
#include "det.cuh"
#else
#include "common.cuh"
#include "det.cuh"
#endif

namespace mfn {

__device__ __forceinline__ void det_warp_max_to(unsigned m, unsigned* __restrict__ out) {
  m = __reduce_max_sync(0xffffffffu, m);
  if ((threadIdx.x & 31) == 0 && m) atomicMax(out, m);
}

// blockDim: a multiple of 32 (every lane reaches the warp reduction)
__global__ void __launch_bounds__(256) det_abs_max_kernel(const float* __restrict__ v, long long n, unsigned* __restrict__ out) {
  unsigned m = 0;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    m = max(m, det_abs_bits(__ldg(v + i)));
  det_warp_max_to(m, out);
}

__global__ void __launch_bounds__(256)
    det_pixel_abs_sum_max_kernel(const float* __restrict__ g, int N, int F, long long HW, unsigned* __restrict__ out) {
  unsigned m = 0;
  const long long total = (long long)N * HW;
  for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < total; p += (long long)gridDim.x * blockDim.x) {
    const long long n = p / HW, pix = p - n * HW;
    const float* gp = g + (size_t)n * F * HW + pix;
    float s = 0.f;
    for (int f = 0; f < F; ++f) s += fabsf(__ldg(gp + (size_t)f * HW));
    m = max(m, det_abs_bits(s));
  }
  det_warp_max_to(m, out);
}

__global__ void __launch_bounds__(256)
    det_fixed_to_float_kernel(const unsigned long long* __restrict__ acc, float* __restrict__ out, long long n,
                              const unsigned* __restrict__ bound, int nb, int fanin_bits) {
  const FixedScale f = det_scale(bound, nb, fanin_bits);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    out[i] += det_from_fixed(acc[i], f);
}

__global__ void __launch_bounds__(256)
    det_ordered_sum_kernel(const float* __restrict__ part, int nparts, long long part_stride, long long elem_stride,
                           float* __restrict__ out, long long n, int accumulate) {
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (long long)gridDim.x * blockDim.x) {
    const float* p = part + e * elem_stride;
    float s = 0.f;
    for (int b = 0; b < nparts; ++b) s += __ldg(p + (size_t)b * part_stride);
    out[e] = accumulate ? out[e] + s : s;
  }
}

}  // namespace mfn

#ifndef MFN_HOST_EMULATION
namespace mfn {

int det_launch_abs_max(const float* v, long long n, unsigned* bound, cudaStream_t st) {
  det_abs_max_kernel<<<grid_for(n, 256), 256, 0, st>>>(v, n, bound);
  return check_launch("det_abs_max_kernel");
}

int det_launch_pixel_abs_sum_max(const float* g, int N, int F, long long HW, unsigned* bound, cudaStream_t st) {
  det_pixel_abs_sum_max_kernel<<<grid_for((long long)N * HW, 256), 256, 0, st>>>(g, N, F, HW, bound);
  return check_launch("det_pixel_abs_sum_max_kernel");
}

int det_launch_fixed_to_float(const unsigned long long* acc, float* out, long long n, const unsigned* bound, int nb,
                              int fanin_bits, cudaStream_t st) {
  det_fixed_to_float_kernel<<<grid_for(n, 256), 256, 0, st>>>(acc, out, n, bound, nb, fanin_bits);
  return check_launch("det_fixed_to_float_kernel");
}

int det_launch_ordered_sum(const float* part, int nparts, long long part_stride, long long elem_stride, float* out,
                           long long n, int accumulate, cudaStream_t st) {
  det_ordered_sum_kernel<<<grid_for(n, 256), 256, 0, st>>>(part, nparts, part_stride, elem_stride, out, n, accumulate);
  return check_launch("det_ordered_sum_kernel");
}

int det_check_workspace(const char* fn, const void* ws, long long bytes, long long need) {
  MFN_REQUIRE(ws, MFN_ERR_INVALID_ARG, "%s: null pointer (det_ws, the deterministic workspace, is required)", fn);
  MFN_REQUIRE(bytes >= need, MFN_ERR_INVALID_ARG, "%s: det_ws holds %lld bytes, the shape needs %lld", fn, bytes, need);
  MFN_REQUIRE(aligned(ws, 16), MFN_ERR_ALIGNMENT, "%s: det_ws must be 16-byte aligned", fn);
  return MFN_OK;
}

}  // namespace mfn
#endif  // !MFN_HOST_EMULATION
