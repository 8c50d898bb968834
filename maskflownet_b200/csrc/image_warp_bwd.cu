// image_warp_bwd.cu -- backward of the image warp for sm_90a: GridGenerator('warp'), BilinearSampler and the fused
// cascade-input builder K5 (forwards in warp_fwd.cu; network/layer.py:8-18, network/MaskFlownet.py:308-313).
//
// One thread per output pixel, like the forwards.  It recomputes the four corners and their weights (sampling.cuh, the same
// code as the forward) and their derivative with respect to the sample position, then walks the channels:
//   position gradient   sum_c grad_out_c * sum_t d wt[t] / d pos * data_c[corner t]     written by the owning thread:
//                       grad_grid, grad_flow_up (and grad_mask_up) use no atomics and are bit-reproducible;
//   data gradient       grad_out_c * wt[t] scattered to the four corners with atomics, ACCUMULATED (the caller zero-fills),
//                       the convention of mfn_deformable_conv_backward; with DET (the *_det entry points) int64
//                       fixed-point sums instead (det.cuh: bound = max |grad_out|, converted by det_fixed_to_float_kernel).
// K5 stops at the up-sampled flow / mask; the transposed Upsample(4) to the quarter-resolution grid is
// mfn_upsample_backward, as for mfn_warp_mask_backward.
//
// The file also builds for the host (MFN_HOST_EMULATION: tests/host_emu/), one thread at a time.
#ifdef MFN_HOST_EMULATION
#include "cuda_shim.h"
#include "sampling.cuh"
#include "det.cuh"
#else
#include "common.cuh"
#include "det.cuh"
#endif

namespace mfn {

// grid[:,0] = (flow[:,0] + x) / ((W-1)/2) - 1, grid[:,1] = (flow[:,1] + y) / ((H-1)/2) - 1
__global__ void gridgen_warp_bwd_kernel(const float* __restrict__ grad_grid, float* __restrict__ grad_flow, int N, int H,
                                        int W) {
  const long long total = (long long)N * H * W;
  const float sx = (float)(W - 1) / 2.f, sy = (float)(H - 1) / 2.f;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const int x = (int)(idx % W), y = (int)((idx / W) % H);
    const long long n = idx / ((long long)W * H);
    const size_t i0 = ((size_t)n * 2) * H * W + (size_t)y * W + x, i1 = i0 + (size_t)H * W;
    grad_flow[i0] = __fdiv_rn(__ldg(grad_grid + i0), sx);
    grad_flow[i1] = __fdiv_rn(__ldg(grad_grid + i1), sy);
  }
}

// Channel walk shared by the sampler and K5: scatters grad_out * wt into grad_data (if given) and returns the position
// gradient (d/dxr, d/dyr).  go / data / gd point at channel 0 of the sample; strides are the channel plane sizes.
// DET: the scatter goes to the fixed-point sums gq (same layout as gd) at scale fsc instead.
template <bool DET>
__device__ __forceinline__ void sample_backward(const float* __restrict__ go, size_t go_plane, const float* __restrict__ data,
                                                float* __restrict__ gd, size_t plane, int C, const int (&off)[4],
                                                const float (&wt)[4], const float (&dwx)[4], const float (&dwy)[4],
                                                bool want_pos, float& gx, float& gy, unsigned long long* __restrict__ gq,
                                                const FixedScale& fsc) {
  float ax = 0.f, ay = 0.f;
  for (int c = 0; c < C; ++c) {
    const float g = __ldg(go + (size_t)c * go_plane);
    if (want_pos) {
      const float* pl = data + (size_t)c * plane;
      float sx = 0.f, sy = 0.f;
#pragma unroll
      for (int t = 0; t < 4; ++t) {
        if (dwx[t] != 0.f || dwy[t] != 0.f) {     // a corner outside the image reads 0
          const float v = __ldg(pl + off[t]);
          sx += dwx[t] * v;
          sy += dwy[t] * v;
        }
      }
      ax += g * sx;
      ay += g * sy;
    }
    if constexpr (DET) {
      if (gq) {
        unsigned long long* qp = gq + (size_t)c * plane;
#pragma unroll
        for (int t = 0; t < 4; ++t)
          if (wt[t] != 0.f) det_scatter(qp + off[t], g * wt[t], fsc);
      }
    } else if (gd) {
      float* gp = gd + (size_t)c * plane;
#pragma unroll
      for (int t = 0; t < 4; ++t)
        if (wt[t] != 0.f) atomicAdd(gp + off[t], g * wt[t]);
    }
  }
  gx = ax;
  gy = ay;
}

template <bool DET>
__device__ __forceinline__ void bilinear_sampler_bwd_body(const float* __restrict__ grad_out, const float* __restrict__ data,
                                            const float* __restrict__ grid, float* __restrict__ grad_data,
                                            float* __restrict__ grad_grid, int N, int C, int H, int W, int OH, int OW,
                                            unsigned long long* __restrict__ gacc, const unsigned* __restrict__ bound,
                                            int fanin_bits) {
  FixedScale fsc{};
  if constexpr (DET) fsc = det_scale(bound, 1, fanin_bits);
  const long long total = (long long)N * OH * OW;
  const size_t oplane = (size_t)OH * OW, plane = (size_t)H * W;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const int x = (int)(idx % OW), y = (int)((idx / OW) % OH);
    const long long n = idx / ((long long)OW * OH);
    const size_t pix = (size_t)y * OW + x;
    const float gx = __ldg(grid + ((size_t)n * 2) * oplane + pix);
    const float gy = __ldg(grid + ((size_t)n * 2 + 1) * oplane + pix);
    // same de-normalisation as bilinear_sampler_kernel: d xr / d gx = (W-1)/2, d yr / d gy = (H-1)/2
    const float xr = (gx + 1.f) * (float)(W - 1) / 2.f, yr = (gy + 1.f) * (float)(H - 1) / 2.f;
    int off[4];
    float wt[4], dwx[4], dwy[4];
    sampler_taps_grad(xr, yr, H, W, off, wt, dwx, dwy);
    float dx, dy;
    sample_backward<DET>(grad_out + (size_t)n * C * oplane + pix, oplane, data + (size_t)n * C * plane,
                         grad_data ? grad_data + (size_t)n * C * plane : nullptr, plane, C, off, wt, dwx, dwy,
                         grad_grid != nullptr, dx, dy, gacc ? gacc + (size_t)n * C * plane : nullptr, fsc);
    if (grad_grid) {
      grad_grid[((size_t)n * 2) * oplane + pix] = dx * ((float)(W - 1) / 2.f);
      grad_grid[((size_t)n * 2 + 1) * oplane + pix] = dy * ((float)(H - 1) / 2.f);
    }
  }
}

// K5 backward: c40[:, c] = sample(im2_c, pix + Upsample(4)(flow_q) * scale) for c < Ci, c40[:, Ci] = sigmoid(Upsample(4)(mask_q)) - 0.5
template <bool DET>
__device__ __forceinline__ void image_warp_concat_bwd_body(const float* __restrict__ grad_c40, const float* __restrict__ im2,
                                             const float* __restrict__ flow_q, const float* __restrict__ mask_q,
                                             float* __restrict__ grad_im2, float* __restrict__ grad_flow_up,
                                             float* __restrict__ grad_mask_up, int N, int Ci, int H, int W, float scale,
                                             unsigned long long* __restrict__ gacc, const unsigned* __restrict__ bound,
                                             int fanin_bits) {
  FixedScale fsc{};
  if constexpr (DET) fsc = det_scale(bound, 1, fanin_bits);
  const int Hq = H / 4, Wq = W / 4;
  const long long total = (long long)N * H * W;
  const size_t plane = (size_t)H * W;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const int x = (int)(idx % W), y = (int)((idx / W) % H);
    const long long n = idx / ((long long)W * H);
    const size_t pix = (size_t)y * W + x;
    const float* gc = grad_c40 + (size_t)n * (Ci + 1) * plane + pix;
    if (grad_im2 || gacc || grad_flow_up) {
      const float* fq = flow_q + (size_t)n * 2 * Hq * Wq;
      const float fy = upsample_at(fq, Hq, Wq, 4, y, x) * scale;
      const float fx = upsample_at(fq + (size_t)Hq * Wq, Hq, Wq, 4, y, x) * scale;
      int off[4];
      float wt[4], dwx[4], dwy[4];
      sampler_taps_grad((float)x + fx, (float)y + fy, H, W, off, wt, dwx, dwy);
      float dx, dy;
      sample_backward<DET>(gc, plane, im2 + (size_t)n * Ci * plane, grad_im2 ? grad_im2 + (size_t)n * Ci * plane : nullptr,
                           plane, Ci, off, wt, dwx, dwy, grad_flow_up != nullptr, dx, dy,
                           gacc ? gacc + (size_t)n * Ci * plane : nullptr, fsc);
      if (grad_flow_up) {   // (y, x) channel order, like flow_q
        grad_flow_up[((size_t)n * 2) * plane + pix] = dy * scale;
        grad_flow_up[((size_t)n * 2 + 1) * plane + pix] = dx * scale;
      }
    }
    if (grad_mask_up) {
      const float s = sigmoidf_(upsample_at(mask_q + (size_t)n * Hq * Wq, Hq, Wq, 4, y, x));
      grad_mask_up[(size_t)n * plane + pix] = __ldg(gc + (size_t)Ci * plane) * (s * (1.f - s));
    }
  }
}

__global__ void bilinear_sampler_bwd_kernel(const float* __restrict__ grad_out, const float* __restrict__ data,
                                            const float* __restrict__ grid, float* __restrict__ grad_data,
                                            float* __restrict__ grad_grid, int N, int C, int H, int W, int OH, int OW) {
  bilinear_sampler_bwd_body<false>(grad_out, data, grid, grad_data, grad_grid, N, C, H, W, OH, OW, nullptr, nullptr, 0);
}

__global__ void bilinear_sampler_bwd_det_kernel(const float* __restrict__ grad_out, const float* __restrict__ data,
                                                const float* __restrict__ grid, float* __restrict__ grad_grid, int N, int C,
                                                int H, int W, int OH, int OW, unsigned long long* __restrict__ gacc,
                                                const unsigned* __restrict__ bound, int fanin_bits) {
  bilinear_sampler_bwd_body<true>(grad_out, data, grid, nullptr, grad_grid, N, C, H, W, OH, OW, gacc, bound, fanin_bits);
}

__global__ void image_warp_concat_bwd_kernel(const float* __restrict__ grad_c40, const float* __restrict__ im2,
                                             const float* __restrict__ flow_q, const float* __restrict__ mask_q,
                                             float* __restrict__ grad_im2, float* __restrict__ grad_flow_up,
                                             float* __restrict__ grad_mask_up, int N, int Ci, int H, int W, float scale) {
  image_warp_concat_bwd_body<false>(grad_c40, im2, flow_q, mask_q, grad_im2, grad_flow_up, grad_mask_up, N, Ci, H, W, scale,
                                    nullptr, nullptr, 0);
}

__global__ void image_warp_concat_bwd_det_kernel(const float* __restrict__ grad_c40, const float* __restrict__ im2,
                                                 const float* __restrict__ flow_q, const float* __restrict__ mask_q,
                                                 float* __restrict__ grad_flow_up, float* __restrict__ grad_mask_up, int N,
                                                 int Ci, int H, int W, float scale, unsigned long long* __restrict__ gacc,
                                                 const unsigned* __restrict__ bound, int fanin_bits) {
  image_warp_concat_bwd_body<true>(grad_c40, im2, flow_q, mask_q, nullptr, grad_flow_up, grad_mask_up, N, Ci, H, W, scale,
                                   gacc, bound, fanin_bits);
}

}  // namespace mfn

#ifndef MFN_HOST_EMULATION
extern "C" int mfn_grid_generator_warp_backward(const float* grad_grid, float* grad_flow, int N, int H, int W, void* stream) {
  using namespace mfn;
  MFN_REQUIRE(grad_grid && grad_flow, MFN_ERR_INVALID_ARG, "mfn_grid_generator_warp_backward: null pointer");
  MFN_REQUIRE(N > 0 && H > 1 && W > 1, MFN_ERR_INVALID_ARG, "mfn_grid_generator_warp_backward: need H, W > 1");
  gridgen_warp_bwd_kernel<<<grid_for((long long)N * H * W, 256), 256, 0, as_stream(stream)>>>(grad_grid, grad_flow, N, H, W);
  return check_launch("gridgen_warp_bwd_kernel");
}

namespace mfn {

// Deterministic workspace of the sampler and K5 (maskflow_b200.h): the bound words, then the int64 sums of the data gradient.
static long long det_sampler_bytes(int N, int C, int H, int W) { return kDetHeaderBytes + 8LL * N * C * H * W; }

// zero the sums and measure the bound (max |grad_out| over the channels that scatter)
static int det_sampler_prologue(void* ws, long long n_acc, const float* go, long long n_go, cudaStream_t st) {
  const cudaError_t ce = cudaMemsetAsync(ws, 0, kDetHeaderBytes + 8 * n_acc, st);
  if (ce != cudaSuccess) return fail((int)ce, "deterministic sampler backward: cudaMemsetAsync: %s", cudaGetErrorString(ce));
  return det_launch_abs_max(go, n_go, static_cast<unsigned*>(ws), st);
}

static unsigned long long* det_acc(void* ws) {
  return reinterpret_cast<unsigned long long*>(static_cast<char*>(ws) + kDetHeaderBytes);
}

static int bilinear_sampler_backward(const float* grad_out, const float* data, const float* grid, float* grad_data,
                                     float* grad_grid, int N, int C, int H, int W, int OH, int OW, void* stream,
                                     void* det_ws, long long det_ws_bytes, bool det) {
  const char* fn = det ? "mfn_bilinear_sampler_backward_det" : "mfn_bilinear_sampler_backward";
  MFN_REQUIRE(grad_out && data && grid, MFN_ERR_INVALID_ARG, "%s: null pointer", fn);
  MFN_REQUIRE(grad_data || grad_grid, MFN_ERR_INVALID_ARG,
              "%s: null pointer (neither grad_data nor grad_grid requested)", fn);
  MFN_REQUIRE(N > 0 && C > 0 && H > 0 && W > 0 && OH > 0 && OW > 0, MFN_ERR_INVALID_ARG, "%s: bad extent", fn);
  cudaStream_t st = as_stream(stream);
  const unsigned blocks = grid_for((long long)N * OH * OW, 256);
  if (!det) {
    bilinear_sampler_bwd_kernel<<<blocks, 256, 0, st>>>(grad_out, data, grid, grad_data, grad_grid, N, C, H, W, OH, OW);
    return check_launch("bilinear_sampler_bwd_kernel");
  }
  int rc = det_check_workspace(fn, det_ws, det_ws_bytes, det_sampler_bytes(N, C, H, W));
  if (rc) return rc;
  const long long n_acc = (long long)N * C * H * W;
  const int fanin_bits = det_bits(4LL * OH * OW);   // every output pixel of the sample, four corners each
  const unsigned* bound = static_cast<const unsigned*>(det_ws);
  unsigned long long* acc = grad_data ? det_acc(det_ws) : nullptr;
  if (grad_data && (rc = det_sampler_prologue(det_ws, n_acc, grad_out, (long long)N * C * OH * OW, st))) return rc;
  bilinear_sampler_bwd_det_kernel<<<blocks, 256, 0, st>>>(grad_out, data, grid, grad_grid, N, C, H, W, OH, OW, acc, bound,
                                                          fanin_bits);
  if ((rc = check_launch("bilinear_sampler_bwd_det_kernel"))) return rc;
  return grad_data ? det_launch_fixed_to_float(acc, grad_data, n_acc, bound, 1, fanin_bits, st) : MFN_OK;
}

static int image_warp_concat_backward(const float* grad_c40, const float* im2, const float* flow_q, const float* mask_q,
                                      float* grad_im2, float* grad_flow_up, float* grad_mask_up, int N, int Ci, int H,
                                      int W, float flow_scale, void* stream, void* det_ws, long long det_ws_bytes,
                                      bool det) {
  const char* fn = det ? "mfn_image_warp_concat_backward_det" : "mfn_image_warp_concat_backward";
  MFN_REQUIRE(grad_c40 && im2 && flow_q && mask_q, MFN_ERR_INVALID_ARG, "%s: null pointer", fn);
  MFN_REQUIRE(grad_im2 || grad_flow_up || grad_mask_up, MFN_ERR_INVALID_ARG, "%s: null pointer (no gradient requested)",
              fn);
  MFN_REQUIRE(N > 0 && Ci > 0 && H > 0 && W > 0 && H % 4 == 0 && W % 4 == 0, MFN_ERR_INVALID_ARG,
              "%s: H and W must be positive multiples of 4", fn);
  cudaStream_t st = as_stream(stream);
  const unsigned blocks = grid_for((long long)N * H * W, 256);
  if (!det) {
    image_warp_concat_bwd_kernel<<<blocks, 256, 0, st>>>(grad_c40, im2, flow_q, mask_q, grad_im2, grad_flow_up,
                                                         grad_mask_up, N, Ci, H, W, flow_scale);
    return check_launch("image_warp_concat_bwd_kernel");
  }
  int rc = det_check_workspace(fn, det_ws, det_ws_bytes, det_sampler_bytes(N, Ci, H, W));
  if (rc) return rc;
  const long long n_acc = (long long)N * Ci * H * W;
  const int fanin_bits = det_bits(4LL * H * W);
  const unsigned* bound = static_cast<const unsigned*>(det_ws);
  unsigned long long* acc = grad_im2 ? det_acc(det_ws) : nullptr;
  // the bound covers all Ci + 1 channels of grad_c40: the mask channel does not scatter, but a larger bound is still one
  if (grad_im2 && (rc = det_sampler_prologue(det_ws, n_acc, grad_c40, (long long)N * (Ci + 1) * H * W, st))) return rc;
  image_warp_concat_bwd_det_kernel<<<blocks, 256, 0, st>>>(grad_c40, im2, flow_q, mask_q, grad_flow_up, grad_mask_up, N,
                                                           Ci, H, W, flow_scale, acc, bound, fanin_bits);
  if ((rc = check_launch("image_warp_concat_bwd_det_kernel"))) return rc;
  return grad_im2 ? det_launch_fixed_to_float(acc, grad_im2, n_acc, bound, 1, fanin_bits, st) : MFN_OK;
}

}  // namespace mfn

extern "C" int mfn_bilinear_sampler_backward(const float* grad_out, const float* data, const float* grid, float* grad_data,
                                             float* grad_grid, int N, int C, int H, int W, int OH, int OW, void* stream) {
  return mfn::bilinear_sampler_backward(grad_out, data, grid, grad_data, grad_grid, N, C, H, W, OH, OW, stream, nullptr, 0,
                                        false);
}

extern "C" int mfn_bilinear_sampler_backward_det(const float* grad_out, const float* data, const float* grid,
                                                 float* grad_data, float* grad_grid, int N, int C, int H, int W, int OH,
                                                 int OW, void* det_ws, long long det_ws_bytes, void* stream) {
  return mfn::bilinear_sampler_backward(grad_out, data, grid, grad_data, grad_grid, N, C, H, W, OH, OW, stream, det_ws,
                                        det_ws_bytes, true);
}

extern "C" int mfn_image_warp_concat_backward(const float* grad_c40, const float* im2, const float* flow_q,
                                              const float* mask_q, float* grad_im2, float* grad_flow_up,
                                              float* grad_mask_up, int N, int Ci, int H, int W, float flow_scale,
                                              void* stream) {
  return mfn::image_warp_concat_backward(grad_c40, im2, flow_q, mask_q, grad_im2, grad_flow_up, grad_mask_up, N, Ci, H, W,
                                         flow_scale, stream, nullptr, 0, false);
}

extern "C" int mfn_image_warp_concat_backward_det(const float* grad_c40, const float* im2, const float* flow_q,
                                                  const float* mask_q, float* grad_im2, float* grad_flow_up,
                                                  float* grad_mask_up, int N, int Ci, int H, int W, float flow_scale,
                                                  void* det_ws, long long det_ws_bytes, void* stream) {
  return mfn::image_warp_concat_backward(grad_c40, im2, flow_q, mask_q, grad_im2, grad_flow_up, grad_mask_up, N, Ci, H, W,
                                         flow_scale, stream, det_ws, det_ws_bytes, true);
}
#endif  // !MFN_HOST_EMULATION
