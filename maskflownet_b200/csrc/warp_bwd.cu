// warp_bwd.cu -- backward of the flow-guided feature warp (K4) for sm_90a.
//
// Serves mfn_deformable_conv_backward and mfn_warp_mask_backward: the gradients that the reference obtains from
// autograd through  F.contrib.DeformableConvolution (network/layer.py:117-124), the `repeat` that builds its offsets
// (network/MaskFlownet.py:230: the nine tap gradients sum into the flow), the sigmoid-mask multiply and the trade-off
// add (:232), and LeakyReLU (:233); triggered at network/pipeline.py:112-113.
//
// Analytic derivative of the forward in warp_fwd.cu:
//   out  = leaky(pre),  pre = conv * sig(m) + tradeoff,  conv[f] = b[f] + sum_k W[f,k] S[k],  S[k] = bilinear sample
//   g_pre = g_out * leaky'(out);  g_tradeoff = g_pre;  g_conv = g_pre * sig(m);  g_m = sig(1-sig) * sum_f g_pre*conv
//   g_b[f] = sum_p g_conv;  g_W[f,k] = sum_p g_conv[f] S[k];  g_S[k] = sum_f W[f,k] g_conv[f]
//   g_x += g_S[k] * (bilinear corner weights)  (scatter);  g_coord = g_S[k] * dS/dcoord;  g_flow = sum_taps g_coord * scale/stride
// Three kernels: warp_bwd_pre (element-wise part), deform_bwd_input (g_S, scatter to g_x, coordinate gradients) and
// deform_bwd_weight (g_W as a pixel-reduction GEMM through shared memory), plus a plane reduction for g_b.
#include "common.cuh"

namespace mfn {

struct AxisG {
  int i0, i1;
  float w0, w1;    // value weights
  float d0, d1;    // d(weight)/d(coordinate)
};

template <int BORDER>
__device__ __forceinline__ AxisG make_axis_g(float c, int n) {
  AxisG a;
  if (BORDER == MFN_BORDER_MXNET15) {
    const bool valid = (c >= 0.f) && (c < (float)n);
    int c0 = (int)floorf(c);
    float l;
    bool collapsed = false;
    if (c0 >= n - 1) {
      c0 = n - 1;
      a.i1 = c0;
      l = 0.f;
      collapsed = true;
    } else {
      a.i1 = c0 + 1;
      l = c - (float)c0;
    }
    a.i0 = c0;
    a.w0 = 1.f - l;
    a.w1 = l;
    a.d0 = collapsed ? 0.f : -1.f;
    a.d1 = collapsed ? 0.f : 1.f;
    if (!valid) {
      a.i0 = a.i1 = 0;
      a.w0 = a.w1 = a.d0 = a.d1 = 0.f;
    }
  } else {
    const bool valid = (c > -1.f) && (c < (float)n);
    const int c0 = (int)floorf(c);
    const float l = c - (float)c0;
    const bool in0 = valid && c0 >= 0, in1 = valid && c0 + 1 <= n - 1;
    a.w0 = in0 ? 1.f - l : 0.f;
    a.w1 = in1 ? l : 0.f;
    a.d0 = in0 ? -1.f : 0.f;
    a.d1 = in1 ? 1.f : 0.f;
    a.i0 = max(min(c0, n - 1), 0);
    a.i1 = max(min(c0 + 1, n - 1), 0);
  }
  return a;
}

// ---------------------------------------------------------------------------------------------------------
// element-wise part: one thread per pixel, loops over the F planes (coalesced per plane)
// ---------------------------------------------------------------------------------------------------------
__global__ void warp_bwd_pre_kernel(const float* __restrict__ gout, const float* __restrict__ out,
                                    const float* __restrict__ conv, const float* __restrict__ mask_up,
                                    float* __restrict__ gconv, float* __restrict__ gtrade,
                                    float* __restrict__ gmask, int N, int F, int H, int W, float slope) {
  const size_t plane = (size_t)H * W;
  const long long total = (long long)N * plane;
  for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < total;
       p += (long long)gridDim.x * blockDim.x) {
    const long long n = p / plane;
    const size_t pix = (size_t)(p - n * plane);
    const float sig = mask_up ? sigmoidf_(__ldg(mask_up + p)) : 1.f;
    float gm = 0.f;
    for (int f = 0; f < F; ++f) {
      const size_t i = ((size_t)n * F + f) * plane + pix;
      float g = __ldg(gout + i);
      if (!(__ldg(out + i) > 0.f)) g *= slope;
      if (gtrade) gtrade[i] = g;
      gconv[i] = g * sig;
      if (gmask) gm = fmaf(g, __ldg(conv + i), gm);
    }
    if (gmask) gmask[p] = gm * sig * (1.f - sig);
  }
}

// sum over (n, pixels) of one plane f:  acc[f] += sum   (one CTA per f)
__global__ void plane_sum_kernel(const float* __restrict__ g, float* __restrict__ acc, int N, int F, int HW) {
  const int f = blockIdx.x;
  float s = 0.f;
  for (int n = 0; n < N; ++n) {
    const float* p = g + ((size_t)n * F + f) * HW;
    for (int i = threadIdx.x; i < HW; i += blockDim.x) s += __ldg(p + i);
  }
  __shared__ float red[32];
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x < 32) {
    s = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : 0.f;
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (threadIdx.x == 0) atomicAdd(acc + f, s);
  }
}

// ---------------------------------------------------------------------------------------------------------
// g_S, scatter into g_x, coordinate gradients.  One thread per pixel; CB input channels (9*CB k values) per pass.
// ---------------------------------------------------------------------------------------------------------
namespace k4 {
constexpr int NT = 256;
constexpr int CB = 4;
constexpr int KB = CB * 9;
constexpr int FT = 32;
}  // namespace k4

template <int BORDER, bool SHARED>
__global__ void __launch_bounds__(k4::NT)
    deform_bwd_input_kernel(const float* __restrict__ gconv, const float* __restrict__ x,
                            const float* __restrict__ offset, const float* __restrict__ flow_up,
                            const float* __restrict__ weight, float* __restrict__ gx, float* __restrict__ gcoord,
                            int N, int C, int H, int W, int F, int Fpad, float flow_scale, float level_stride) {
  using namespace k4;
  extern __shared__ __align__(16) float Wt[];  // [KB][Fpad]
  const int tid = threadIdx.x;
  const size_t plane = (size_t)H * W;
  const long long total = (long long)N * plane;
  const long long p = (long long)blockIdx.x * NT + tid;
  const bool live = p < total;
  int n = 0, y = 0, xq = 0;
  if (live) {
    xq = (int)(p % W);
    y = (int)((p / W) % H);
    n = (int)(p / plane);
  }
  const size_t pix = (size_t)y * W + xq;

  AxisG ah[3], aw[3];
  if (SHARED && live) {
    const float fy = __ldg(flow_up + ((size_t)n * 2) * plane + pix);
    const float fx = __ldg(flow_up + ((size_t)n * 2 + 1) * plane + pix);
    const float dy = __fdiv_rn(__fmul_rn(fy, flow_scale), level_stride);
    const float dx = __fdiv_rn(__fmul_rn(fx, flow_scale), level_stride);
#pragma unroll
    for (int i = 0; i < 3; ++i) {
      ah[i] = make_axis_g<BORDER>((float)(y - 1 + i) + dy, H);
      aw[i] = make_axis_g<BORDER>((float)(xq - 1 + i) + dx, W);
    }
  }
  float gdy = 0.f, gdx = 0.f;     // SHARED: summed over taps
  float gtap[SHARED ? 1 : 18];    // per-tap coordinate gradients otherwise
  if (!SHARED) {
#pragma unroll
    for (int i = 0; i < 18; ++i) gtap[i] = 0.f;
  }

  const float* gc = gconv + (size_t)n * F * plane + pix;
  const float* xn = x + (size_t)n * C * plane;
  float* gxn = gx ? gx + (size_t)n * C * plane : nullptr;
  const float* offn = SHARED ? nullptr : offset + (size_t)n * 18 * plane + pix;

  for (int c0 = 0; c0 < C; c0 += CB) {
    __syncthreads();
    for (int e = tid; e < KB * Fpad; e += NT) {
      const int k = e % KB, f = e / KB;
      const int c = c0 + k / 9;
      float v = 0.f;
      if (f < F && c < C) v = __ldg(weight + ((size_t)f * C + c0) * 9 + k);
      Wt[k * Fpad + f] = v;
    }
    __syncthreads();
    if (!live) continue;
    float gS[KB];
#pragma unroll
    for (int k = 0; k < KB; ++k) gS[k] = 0.f;
    for (int f0 = 0; f0 < F; f0 += FT) {
      float g[FT];
#pragma unroll
      for (int f = 0; f < FT; ++f) g[f] = (f0 + f < F) ? __ldg(gc + (size_t)(f0 + f) * plane) : 0.f;
#pragma unroll
      for (int k = 0; k < KB; ++k) {
        const float4* wrow = reinterpret_cast<const float4*>(Wt + k * Fpad + f0);
        float s = gS[k];
#pragma unroll
        for (int fq = 0; fq < FT / 4; ++fq) {
          const float4 w4 = wrow[fq];
          s = fmaf(w4.x, g[4 * fq + 0], s);
          s = fmaf(w4.y, g[4 * fq + 1], s);
          s = fmaf(w4.z, g[4 * fq + 2], s);
          s = fmaf(w4.w, g[4 * fq + 3], s);
        }
        gS[k] = s;
      }
    }
    const int cend = min(CB, C - c0);
#pragma unroll
    for (int tap = 0; tap < 9; ++tap) {
      const int ti = tap / 3, tj = tap - 3 * ti;
      AxisG hA, wA;
      if (SHARED) {
        hA = ah[ti];
        wA = aw[tj];
      } else {
        hA = make_axis_g<BORDER>((float)(y - 1 + ti) + __ldg(offn + (size_t)(2 * tap) * plane), H);
        wA = make_axis_g<BORDER>((float)(xq - 1 + tj) + __ldg(offn + (size_t)(2 * tap + 1) * plane), W);
      }
      const int o00 = hA.i0 * W + wA.i0, o01 = hA.i0 * W + wA.i1, o10 = hA.i1 * W + wA.i0, o11 = hA.i1 * W + wA.i1;
      const float w00 = hA.w0 * wA.w0, w01 = hA.w0 * wA.w1, w10 = hA.w1 * wA.w0, w11 = hA.w1 * wA.w1;
      float th = 0.f, tw = 0.f;
#pragma unroll
      for (int cc = 0; cc < CB; ++cc) {
        if (cc >= cend) break;
        const float gs = gS[cc * 9 + tap];
        const float* pl = xn + (size_t)(c0 + cc) * plane;
        const float v00 = __ldg(pl + o00), v01 = __ldg(pl + o01), v10 = __ldg(pl + o10), v11 = __ldg(pl + o11);
        // dS/dh = d0*(ww0 v00 + ww1 v01) + d1*(ww0 v10 + ww1 v11);  dS/dw = wh0*(dw0 v00 + dw1 v01) + wh1*(dw0 v10 + dw1 v11)
        th = fmaf(gs, hA.d0 * (wA.w0 * v00 + wA.w1 * v01) + hA.d1 * (wA.w0 * v10 + wA.w1 * v11), th);
        tw = fmaf(gs, hA.w0 * (wA.d0 * v00 + wA.d1 * v01) + hA.w1 * (wA.d0 * v10 + wA.d1 * v11), tw);
        if (gxn) {
          float* gp = gxn + (size_t)(c0 + cc) * plane;
          if (w00 != 0.f) atomicAdd(gp + o00, gs * w00);
          if (w01 != 0.f) atomicAdd(gp + o01, gs * w01);
          if (w10 != 0.f) atomicAdd(gp + o10, gs * w10);
          if (w11 != 0.f) atomicAdd(gp + o11, gs * w11);
        }
      }
      if (SHARED) {
        gdy += th;
        gdx += tw;
      } else {
        gtap[2 * tap] += th;
        gtap[2 * tap + 1] += tw;
      }
    }
  }
  if (!live || !gcoord) return;
  if (SHARED) {
    const float s = flow_scale / level_stride;
    gcoord[((size_t)n * 2) * plane + pix] = gdy * s;
    gcoord[((size_t)n * 2 + 1) * plane + pix] = gdx * s;
  } else {
#pragma unroll
    for (int i = 0; i < 18; ++i) gcoord[((size_t)n * 18 + i) * plane + pix] = gtap[i];
  }
}

// ---------------------------------------------------------------------------------------------------------
// g_W[f][c][tap] += sum_p gconv[f][p] * S[p][c][tap].  CTA = 128 pixels; per (channel block, f tile): every thread
// samples its pixel into shared memory, then the CTA contracts the 128-pixel axis and issues one atomic per element.
// ---------------------------------------------------------------------------------------------------------
namespace k4w {
constexpr int PX = 128;   // pixels per CTA (= threads)
constexpr int CB = 4, KB = CB * 9, FT = 32;
}  // namespace k4w

template <int BORDER, bool SHARED>
__global__ void __launch_bounds__(k4w::PX)
    deform_bwd_weight_kernel(const float* __restrict__ gconv, const float* __restrict__ x,
                             const float* __restrict__ offset, const float* __restrict__ flow_up,
                             float* __restrict__ gw, int N, int C, int H, int W, int F, float flow_scale,
                             float level_stride) {
  using namespace k4w;
  __shared__ float Ss[PX][KB + 1];
  __shared__ float Gs[PX][FT + 1];
  const int tid = threadIdx.x;
  const size_t plane = (size_t)H * W;
  const long long total = (long long)N * plane;
  const long long p = (long long)blockIdx.x * PX + tid;
  const bool live = p < total;
  int n = 0, y = 0, xq = 0;
  if (live) {
    xq = (int)(p % W);
    y = (int)((p / W) % H);
    n = (int)(p / plane);
  }
  const size_t pix = (size_t)y * W + xq;
  AxisG ah[3], aw[3];
  if (SHARED && live) {
    const float fy = __ldg(flow_up + ((size_t)n * 2) * plane + pix);
    const float fx = __ldg(flow_up + ((size_t)n * 2 + 1) * plane + pix);
    const float dy = __fdiv_rn(__fmul_rn(fy, flow_scale), level_stride);
    const float dx = __fdiv_rn(__fmul_rn(fx, flow_scale), level_stride);
#pragma unroll
    for (int i = 0; i < 3; ++i) {
      ah[i] = make_axis_g<BORDER>((float)(y - 1 + i) + dy, H);
      aw[i] = make_axis_g<BORDER>((float)(xq - 1 + i) + dx, W);
    }
  }
  const float* xn = x + (size_t)n * C * plane;
  const float* offn = SHARED ? nullptr : offset + (size_t)n * 18 * plane + pix;
  const float* gc = gconv + (size_t)n * F * plane + pix;

  for (int c0 = 0; c0 < C; c0 += CB) {
    __syncthreads();
    // samples of this pixel for channels c0..c0+CB
    for (int tap = 0; tap < 9; ++tap) {
      const int ti = tap / 3, tj = tap - 3 * ti;
      AxisG hA, wA;
      if (live) {
        if (SHARED) {
          hA = ah[ti];
          wA = aw[tj];
        } else {
          hA = make_axis_g<BORDER>((float)(y - 1 + ti) + __ldg(offn + (size_t)(2 * tap) * plane), H);
          wA = make_axis_g<BORDER>((float)(xq - 1 + tj) + __ldg(offn + (size_t)(2 * tap + 1) * plane), W);
        }
      }
      for (int cc = 0; cc < CB; ++cc) {
        float s = 0.f;
        if (live && c0 + cc < C) {
          const float* pl = xn + (size_t)(c0 + cc) * plane;
          s = hA.w0 * wA.w0 * __ldg(pl + hA.i0 * W + wA.i0) + hA.w0 * wA.w1 * __ldg(pl + hA.i0 * W + wA.i1) +
              hA.w1 * wA.w0 * __ldg(pl + hA.i1 * W + wA.i0) + hA.w1 * wA.w1 * __ldg(pl + hA.i1 * W + wA.i1);
        }
        Ss[tid][cc * 9 + tap] = s;
      }
    }
    for (int f0 = 0; f0 < F; f0 += FT) {
      __syncthreads();  // Ss complete (first pass) / previous contraction finished reading Gs
      for (int f = 0; f < FT; ++f) Gs[tid][f] = (live && f0 + f < F) ? __ldg(gc + (size_t)(f0 + f) * plane) : 0.f;
      __syncthreads();
      // 32 x 36 outputs over 128 threads: thread -> (f = tid % 32, k = tid / 32 + 4*i), i = 0..8
      const int f = tid & 31, kb = tid >> 5;
      float acc[9];
#pragma unroll
      for (int i = 0; i < 9; ++i) acc[i] = 0.f;
      for (int q = 0; q < PX; ++q) {
        const float g = Gs[q][f];
#pragma unroll
        for (int i = 0; i < 9; ++i) acc[i] = fmaf(g, Ss[q][kb + 4 * i], acc[i]);
      }
      if (f0 + f < F) {
#pragma unroll
        for (int i = 0; i < 9; ++i) {
          const int k = kb + 4 * i, c = c0 + k / 9;
          if (c < C && acc[i] != 0.f) atomicAdd(gw + ((size_t)(f0 + f) * C + c) * 9 + (k % 9), acc[i]);
        }
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------------------
template <int BORDER, bool SHARED>
static int launch_deform_bwd(const float* gconv, const float* x, const float* offset, const float* flow_up,
                             const float* weight, float* gx, float* gcoord, float* gw, float* gb, int N, int C, int H,
                             int W, int F, float fs, float ls, cudaStream_t st) {
  const long long total = (long long)N * H * W;
  if (gx || gcoord) {
    const int Fpad = ((F + k4::FT - 1) / k4::FT) * k4::FT;
    const int smem = (int)sizeof(float) * k4::KB * Fpad;
    cudaFuncSetAttribute(deform_bwd_input_kernel<BORDER, SHARED>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    const unsigned grid = (unsigned)((total + k4::NT - 1) / k4::NT);
    deform_bwd_input_kernel<BORDER, SHARED><<<grid, k4::NT, smem, st>>>(gconv, x, offset, flow_up, weight, gx, gcoord,
                                                                        N, C, H, W, F, Fpad, fs, ls);
    const int rc = check_launch("deform_bwd_input_kernel");
    if (rc) return rc;
  }
  if (gw) {
    const unsigned grid = (unsigned)((total + k4w::PX - 1) / k4w::PX);
    deform_bwd_weight_kernel<BORDER, SHARED><<<grid, k4w::PX, 0, st>>>(gconv, x, offset, flow_up, gw, N, C, H, W, F,
                                                                       fs, ls);
    const int rc = check_launch("deform_bwd_weight_kernel");
    if (rc) return rc;
  }
  if (gb) {
    plane_sum_kernel<<<F, 256, 0, st>>>(gconv, gb, N, F, H * W);
    return check_launch("plane_sum_kernel");
  }
  return MFN_OK;
}

}  // namespace mfn

extern "C" int mfn_deformable_conv_backward(const float* grad_out, const float* data, const float* offset,
                                            const float* weight, float* grad_data, float* grad_offset,
                                            float* grad_weight, float* grad_bias, int N, int C, int H, int W, int F,
                                            int border_mode, void* stream) {
  using namespace mfn;
  MFN_REQUIRE(grad_out && data && offset && weight, MFN_ERR_INVALID_ARG, "mfn_deformable_conv_backward: null pointer");
  MFN_REQUIRE(N > 0 && C > 0 && H > 0 && W > 0 && F > 0, MFN_ERR_INVALID_ARG,
              "mfn_deformable_conv_backward: non-positive extent");
  MFN_REQUIRE(border_mode == MFN_BORDER_MXNET15 || border_mode == MFN_BORDER_ZERO_CORNER, MFN_ERR_INVALID_ARG,
              "mfn_deformable_conv_backward: unknown border_mode %d", border_mode);
  MFN_REQUIRE(F <= 1024, MFN_ERR_UNSUPPORTED, "mfn_deformable_conv_backward: F > 1024 not supported");
  cudaStream_t st = as_stream(stream);
  if (border_mode == MFN_BORDER_MXNET15)
    return launch_deform_bwd<MFN_BORDER_MXNET15, false>(grad_out, data, offset, nullptr, weight, grad_data,
                                                        grad_offset, grad_weight, grad_bias, N, C, H, W, F, 0.f, 1.f,
                                                        st);
  return launch_deform_bwd<MFN_BORDER_ZERO_CORNER, false>(grad_out, data, offset, nullptr, weight, grad_data,
                                                          grad_offset, grad_weight, grad_bias, N, C, H, W, F, 0.f, 1.f,
                                                          st);
}

extern "C" int mfn_warp_mask_backward(const float* grad_out, const float* out, const float* conv_out, const float* x,
                                      const float* flow_up, const float* mask_up, const float* weight, float* grad_x,
                                      float* grad_flow_up, float* grad_mask_up, float* grad_weight, float* grad_bias,
                                      float* grad_tradeoff, float* grad_conv_ws, int N, int C, int H, int W, int F,
                                      float flow_scale, float level_stride, float leaky_slope, int border_mode,
                                      void* stream) {
  using namespace mfn;
  MFN_REQUIRE(grad_out && out && x && flow_up && weight && grad_conv_ws, MFN_ERR_INVALID_ARG,
              "mfn_warp_mask_backward: null pointer (grad_conv_ws, an (N,F,H,W) workspace, is required)");
  MFN_REQUIRE(!grad_mask_up || (mask_up && conv_out), MFN_ERR_INVALID_ARG,
              "mfn_warp_mask_backward: grad_mask_up needs mask_up and conv_out");
  MFN_REQUIRE(N > 0 && C > 0 && H > 0 && W > 0 && F > 0 && level_stride > 0.f, MFN_ERR_INVALID_ARG,
              "mfn_warp_mask_backward: bad extent");
  MFN_REQUIRE(border_mode == MFN_BORDER_MXNET15 || border_mode == MFN_BORDER_ZERO_CORNER, MFN_ERR_INVALID_ARG,
              "mfn_warp_mask_backward: unknown border_mode %d", border_mode);
  MFN_REQUIRE(F <= 1024, MFN_ERR_UNSUPPORTED, "mfn_warp_mask_backward: F > 1024 not supported");
  cudaStream_t st = as_stream(stream);
  const long long total = (long long)N * H * W;
  long long blocks = (total + 255) / 256;
  if (blocks > kNumSMs * 16) blocks = kNumSMs * 16;
  warp_bwd_pre_kernel<<<(unsigned)blocks, 256, 0, st>>>(grad_out, out, conv_out, mask_up, grad_conv_ws, grad_tradeoff,
                                                        grad_mask_up, N, F, H, W, leaky_slope);
  int rc = check_launch("warp_bwd_pre_kernel");
  if (rc) return rc;
  if (border_mode == MFN_BORDER_MXNET15)
    return launch_deform_bwd<MFN_BORDER_MXNET15, true>(grad_conv_ws, x, nullptr, flow_up, weight, grad_x, grad_flow_up,
                                                       grad_weight, grad_bias, N, C, H, W, F, flow_scale, level_stride,
                                                       st);
  return launch_deform_bwd<MFN_BORDER_ZERO_CORNER, true>(grad_conv_ws, x, nullptr, flow_up, weight, grad_x,
                                                         grad_flow_up, grad_weight, grad_bias, N, C, H, W, F,
                                                         flow_scale, level_stride, st);
}
