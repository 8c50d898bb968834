// sampling.cuh -- interpolation arithmetic shared by the forward and backward warp kernels: the Upsample(f) taps, the
// sigmoid of the occlusion mask, and the four-corner taps of BilinearSampler with their derivative with respect to the
// sample position.  Device functions only and no CUDA runtime header, so that the host emulation of the element-wise
// kernels (MFN_HOST_EMULATION, tests/host_emu/cuda_shim.h) compiles the same arithmetic.
#pragma once

namespace mfn {

__device__ __forceinline__ float sigmoidf_(float v) { return 1.f / (1.f + __expf(-v)); }

// Upsample(f) taps along one axis (network/MaskFlownet.py:35-62): output index o = f*i + r reads
// in[i]*(1-r/f) + in[min(i+1, n-1)]*(r/f).
__device__ __forceinline__ void upsample_taps(int o, int f, int n, int& i0, int& i1, float& w1) {
  i0 = o / f;
  const int r = o - i0 * f;
  i1 = min(i0 + 1, n - 1);
  w1 = (float)r / (float)f;
}

__device__ __forceinline__ float upsample_at(const float* __restrict__ plane, int Hc, int Wc, int f,
                                             int y, int x) {
  int y0, y1, x0, x1;
  float wy, wx;
  upsample_taps(y, f, Hc, y0, y1, wy);
  upsample_taps(x, f, Wc, x0, x1, wx);
  const float a = __ldg(plane + (size_t)y0 * Wc + x0), b = __ldg(plane + (size_t)y0 * Wc + x1);
  const float c = __ldg(plane + (size_t)y1 * Wc + x0), d = __ldg(plane + (size_t)y1 * Wc + x1);
  const float top = a + (b - a) * wx, bot = c + (d - c) * wx;
  return top + (bot - top) * wy;
}

// BilinearSampler taps at the real position (xr, yr) of an H x W plane (network/layer.py:18): corner t = 2*dy + dx of the
// cell whose top-left corner is (floor(yr), floor(xr)).  off[t] is clamped into the plane; a corner outside the plane has
// weight 0 (it reads 0 and receives no data gradient).  With GRAD, dwx[t] = d wt[t] / d xr and dwy[t] = d wt[t] / d yr
// under the same per-corner validity: at lattice points this is the derivative from the floor side, as in MXNet's
// BilinearSamplerBackward and torch's grid_sample backward.
template <bool GRAD>
__device__ __forceinline__ void sampler_corners(float xr, float yr, int H, int W, int (&off)[4], float (&wt)[4],
                                                float (&dwx)[4], float (&dwy)[4]) {
  const int x0 = (int)floorf(xr), y0 = (int)floorf(yr);
  const float wx0 = 1.f - (xr - (float)x0), wy0 = 1.f - (yr - (float)y0);
  const float wx1 = 1.f - wx0, wy1 = 1.f - wy0;
  const bool xin0 = x0 >= 0 && x0 <= W - 1, xin1 = x0 + 1 >= 0 && x0 + 1 <= W - 1;
  const bool yin0 = y0 >= 0 && y0 <= H - 1, yin1 = y0 + 1 >= 0 && y0 + 1 <= H - 1;
  const int xc0 = max(min(x0, W - 1), 0), xc1 = max(min(x0 + 1, W - 1), 0);
  const int yc0 = max(min(y0, H - 1), 0), yc1 = max(min(y0 + 1, H - 1), 0);
  off[0] = yc0 * W + xc0;
  off[1] = yc0 * W + xc1;
  off[2] = yc1 * W + xc0;
  off[3] = yc1 * W + xc1;
  wt[0] = (xin0 && yin0) ? wy0 * wx0 : 0.f;
  wt[1] = (xin1 && yin0) ? wy0 * wx1 : 0.f;
  wt[2] = (xin0 && yin1) ? wy1 * wx0 : 0.f;
  wt[3] = (xin1 && yin1) ? wy1 * wx1 : 0.f;
  if (GRAD) {
    dwx[0] = (xin0 && yin0) ? -wy0 : 0.f;
    dwx[1] = (xin1 && yin0) ? wy0 : 0.f;
    dwx[2] = (xin0 && yin1) ? -wy1 : 0.f;
    dwx[3] = (xin1 && yin1) ? wy1 : 0.f;
    dwy[0] = (xin0 && yin0) ? -wx0 : 0.f;
    dwy[1] = (xin1 && yin0) ? -wx1 : 0.f;
    dwy[2] = (xin0 && yin1) ? wx0 : 0.f;
    dwy[3] = (xin1 && yin1) ? wx1 : 0.f;
  }
}

__device__ __forceinline__ void sampler_taps(float xr, float yr, int H, int W, int (&off)[4], float (&wt)[4]) {
  float unused_x[4], unused_y[4];
  sampler_corners<false>(xr, yr, H, W, off, wt, unused_x, unused_y);
}

__device__ __forceinline__ void sampler_taps_grad(float xr, float yr, int H, int W, int (&off)[4], float (&wt)[4],
                                                  float (&dwx)[4], float (&dwy)[4]) {
  sampler_corners<true>(xr, yr, H, W, off, wt, dwx, dwy);
}

}  // namespace mfn
