// warp_fwd.cu -- flow-guided feature warp forward kernels (K3), Upsample, GridGenerator/BilinearSampler and the
// fused cascade-input builder (K5) for sm_90a.  The image warp's backward kernels are in image_warp_bwd.cu.
//
// K3 serves two entry points with one kernel template:
//   mfn_deformable_conv_forward  F.contrib.DeformableConvolution(x, offset, weight[, bias])   network/layer.py:117-124
//   mfn_warp_mask_forward        Upsample(2)(flow/mask) + deformable conv with all 9 tap offsets = flow*scale/stride
//                                + * sigmoid(mask) + trade-off + LeakyReLU                  network/MaskFlownet.py:228-233
//
// Formulation: out[p, f] = sum_{c, tap} S[p, c, tap] * W[f, c, tap] with S the bilinear samples (an implicit
// im2col that never touches HBM; MXNet materialises it, 9x the input).  One thread owns one output pixel and FT
// output channels: it gathers its own samples into registers, and reads the weight chunk from shared memory as
// warp-wide broadcasts, so shared-memory bandwidth is not the limiter and every global store is a coalesced row.
#include "common.cuh"

namespace mfn {

namespace k3 {
constexpr int CC = 8;          // input channels per weight chunk
constexpr int KC = CC * 9;     // k values per chunk
}  // namespace k3

// One axis of a bilinear tap with validity folded into the weights:
//   value = sum_a w[a] * data[idx[a]];  d(value)/d(coord) = sum_a dw[a] * data[idx[a]]
struct Axis {
  int i0, i1;
  float w0, w1;
};

template <int BORDER>
__device__ __forceinline__ Axis make_axis(float c, int n) {
  Axis a;
  if (BORDER == MFN_BORDER_MXNET15) {
    const bool valid = (c >= 0.f) && (c < (float)n);
    int c0 = (int)floorf(c);
    float l;
    if (c0 >= n - 1) {
      c0 = n - 1;
      a.i1 = c0;
      l = 0.f;
    } else {
      a.i1 = c0 + 1;
      l = c - (float)c0;
    }
    a.i0 = c0;
    a.w0 = 1.f - l;
    a.w1 = l;
    if (!valid) {
      a.i0 = a.i1 = 0;
      a.w0 = a.w1 = 0.f;
    }
  } else {
    const bool valid = (c > -1.f) && (c < (float)n);
    const int c0 = (int)floorf(c);
    const float l = c - (float)c0;
    a.w0 = (valid && c0 >= 0) ? 1.f - l : 0.f;
    a.w1 = (valid && c0 + 1 <= n - 1) ? l : 0.f;
    a.i0 = max(min(c0, n - 1), 0);
    a.i1 = max(min(c0 + 1, n - 1), 0);
  }
  return a;
}

// Pixels whose nine taps all sample strictly inside the image (both border rules reduce to plain bilinear there): the
// warped centre lies in [1, H-2] x [1, W-2].  Pixels whose nine taps all fall outside contribute a zero convolution.
__device__ __forceinline__ bool warp_interior(float h0, float w0, int H, int W) {
  return h0 >= 1.f && h0 <= (float)(H - 2) && w0 >= 1.f && w0 <= (float)(W - 2);
}
__device__ __forceinline__ bool warp_far_outside(float h0, float w0, int H, int W) {
  return h0 <= -2.f || h0 >= (float)(H + 1) || w0 <= -2.f || w0 >= (float)(W + 1);
}

// SHARED: all nine taps use the same (dy, dx) (fused warp); otherwise per-tap offsets from `offset` (N,18,H,W).
// FUSED epilogue operands (mask / tradeoff / conv_out / flow outputs) are only used when SHARED.
// NT = threads (= pixels) per CTA: 256 for the big levels, 128 / 64 for the small ones so that the grid still covers the GPU
template <int NT, int FT, int BORDER, bool SHARED>
__global__ void __launch_bounds__(NT, 512 / NT)
    deform_fwd_kernel(const float* __restrict__ x, const float* __restrict__ offset,
                      const float* __restrict__ flow_c, const float* __restrict__ mask_c,
                      const float* __restrict__ weight, const float* __restrict__ bias,
                      const float* __restrict__ tradeoff, float* __restrict__ out, float* __restrict__ flow_up_out,
                      float* __restrict__ mask_up_out, float* __restrict__ conv_out, int N, int C, int H, int W,
                      int F, int up, float flow_scale, float level_stride, float slope,
                      const int* __restrict__ pix_list, const int* __restrict__ pix_count) {
  using namespace k3;
  __shared__ __align__(16) float Wt[KC * FT];  // [k][f], f-quads XOR-swizzled by (k & 7)

  const int tid = threadIdx.x;
  const long long total = (long long)N * H * W;
  // pix_list: this launch serves only the listed pixels (the border frame left over by warp_resample_kernel); the grid is
  // sized for the worst case, CTAs beyond the list leave at once
  long long p = (long long)blockIdx.x * NT + tid;
  bool live = p < total;
  if (pix_list) {
    const int cnt = *pix_count;
    if ((long long)blockIdx.x * NT >= cnt) return;
    live = p < cnt;
    p = live ? pix_list[p] : 0;
  }
  const int f0 = blockIdx.y * FT;
  const size_t plane = (size_t)H * W;

  int n = 0, y = 0, xq = 0;
  if (live) {
    xq = (int)(p % W);
    y = (int)((p / W) % H);
    n = (int)(p / plane);
  }

  Axis ah[3], aw[3];
  float mask_v = 0.f;
  if (SHARED && live) {
    const int Hc = H / up, Wc = W / up;
    const float* fc = flow_c + (size_t)n * 2 * Hc * Wc;
    const float fy = upsample_at(fc, Hc, Wc, up, y, xq);
    const float fx = upsample_at(fc + (size_t)Hc * Wc, Hc, Wc, up, y, xq);
    if (mask_c) mask_v = upsample_at(mask_c + (size_t)n * Hc * Wc, Hc, Wc, up, y, xq);
    if (blockIdx.y == 0) {
      if (flow_up_out) {
        flow_up_out[((size_t)n * 2 + 0) * plane + (size_t)y * W + xq] = fy;
        flow_up_out[((size_t)n * 2 + 1) * plane + (size_t)y * W + xq] = fx;
      }
      if (mask_up_out && mask_c) mask_up_out[(size_t)n * plane + (size_t)y * W + xq] = mask_v;
    }
    // offsets exactly as the reference rounds them: (flow * scale) / stride   (MaskFlownet.py:230)
    const float dy = __fdiv_rn(__fmul_rn(fy, flow_scale), level_stride);
    const float dx = __fdiv_rn(__fmul_rn(fx, flow_scale), level_stride);
#pragma unroll
    for (int i = 0; i < 3; ++i) {
      ah[i] = make_axis<BORDER>((float)(y - 1 + i) + dy, H);
      aw[i] = make_axis<BORDER>((float)(xq - 1 + i) + dx, W);
    }
  }

  float acc[FT];
#pragma unroll
  for (int f = 0; f < FT; ++f) acc[f] = 0.f;

  const float* xn = x + (size_t)n * C * plane;
  const float* offn = SHARED ? nullptr : offset + (size_t)n * 18 * plane + (size_t)y * W + xq;

  for (int c0 = 0; c0 < C; c0 += CC) {
    __syncthreads();
    // weight chunk: W[f][c0..c0+CC)[9] is contiguous in k for each f -> coalesced reads along k
    for (int e = tid; e < KC * FT; e += NT) {
      const int k = e % KC, f = e / KC;
      const int c = c0 + k / 9;
      float v = 0.f;
      if (f0 + f < F && c < C) v = __ldg(weight + ((size_t)(f0 + f) * C + c0) * 9 + k);
      Wt[k * FT + ((((f >> 2) ^ (k & 7)) << 2) | (f & 3))] = v;
    }
    __syncthreads();
    if (!live) continue;
#pragma unroll 1
    for (int tap = 0; tap < 9; ++tap) {
      const int ti = tap / 3, tj = tap - 3 * ti;
      Axis hA, wA;
      if (SHARED) {  // register selects instead of dynamic indexing (keeps ah/aw out of local memory)
        hA = ti == 0 ? ah[0] : (ti == 1 ? ah[1] : ah[2]);
        wA = tj == 0 ? aw[0] : (tj == 1 ? aw[1] : aw[2]);
      } else {
        const float oy = __ldg(offn + (size_t)(2 * tap) * plane);
        const float ox = __ldg(offn + (size_t)(2 * tap + 1) * plane);
        hA = make_axis<BORDER>((float)(y - 1 + ti) + oy, H);
        wA = make_axis<BORDER>((float)(xq - 1 + tj) + ox, W);
      }
      const float w00 = hA.w0 * wA.w0, w01 = hA.w0 * wA.w1, w10 = hA.w1 * wA.w0, w11 = hA.w1 * wA.w1;
      const int o00 = hA.i0 * W + wA.i0, o01 = hA.i0 * W + wA.i1, o10 = hA.i1 * W + wA.i0, o11 = hA.i1 * W + wA.i1;
      const bool any = (w00 != 0.f) || (w01 != 0.f) || (w10 != 0.f) || (w11 != 0.f);
      const int cend = min(CC, C - c0);
      for (int cc = 0; cc < cend; ++cc) {
        float s = 0.f;
        if (any) {
          const float* pl = xn + (size_t)(c0 + cc) * plane;
          // same association as the oracle: ((w00*v00 + w01*v01) + w10*v10) + w11*v11
          s = w00 * __ldg(pl + o00) + w01 * __ldg(pl + o01) + w10 * __ldg(pl + o10) + w11 * __ldg(pl + o11);
        }
        const int k = cc * 9 + tap;
        const float4* wrow = reinterpret_cast<const float4*>(Wt + k * FT);
#pragma unroll
        for (int fq = 0; fq < FT / 4; ++fq) {
          const float4 w4 = wrow[fq ^ (k & 7)];
          acc[4 * fq + 0] = fmaf(s, w4.x, acc[4 * fq + 0]);
          acc[4 * fq + 1] = fmaf(s, w4.y, acc[4 * fq + 1]);
          acc[4 * fq + 2] = fmaf(s, w4.z, acc[4 * fq + 2]);
          acc[4 * fq + 3] = fmaf(s, w4.w, acc[4 * fq + 3]);
        }
      }
    }
  }
  if (!live) return;
  const float sig = (SHARED && mask_c) ? sigmoidf_(mask_v) : 1.f;
  const size_t pix = (size_t)y * W + xq;
#pragma unroll
  for (int f = 0; f < FT; ++f) {
    if (f0 + f >= F) break;
    float v = acc[f];
    if (bias) v += __ldg(bias + f0 + f);
    const size_t oi = ((size_t)n * F + f0 + f) * plane + pix;
    if (SHARED) {
      if (conv_out) conv_out[oi] = v;
      v *= sig;
      if (tradeoff) v += __ldg(tradeoff + oi);
      v = leaky(v, slope);
    }
    out[oi] = v;
  }
}

// ---------------------------------------------------------------------------------------------------------
// Upsample(f) forward / backward (network/MaskFlownet.py:35-62)
// ---------------------------------------------------------------------------------------------------------
// One block row per output row (blockIdx.y = plane * OH + y, no 64-bit index arithmetic per element), four consecutive
// output pixels per thread: row taps once, 16-byte stores when the row is aligned.
__global__ void upsample_fwd_kernel(const float* __restrict__ in, float* __restrict__ out, int planes, int H, int W,
                                    int f, float scale) {
  const int OH = H * f, OW = W * f;
  for (long long row = blockIdx.y; row < (long long)planes * OH; row += gridDim.y) {
    const int pl = (int)(row / OH), y = (int)(row - (long long)pl * OH);
    int y0, y1;
    float wy;
    upsample_taps(y, f, H, y0, y1, wy);
    const float* r0 = in + ((size_t)pl * H + y0) * W;
    const float* r1 = in + ((size_t)pl * H + y1) * W;
    float* orow = out + (size_t)row * OW;
    const bool vec = (OW & 3) == 0 && ((reinterpret_cast<size_t>(orow) & 15) == 0);
    for (int x4 = 4 * (blockIdx.x * blockDim.x + threadIdx.x); x4 < OW; x4 += 4 * gridDim.x * blockDim.x) {
      float v[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const int x = min(x4 + k, OW - 1);
        const int x0 = x / f, x1 = min(x0 + 1, W - 1);
        const float wx = (float)(x - x0 * f) / (float)f;   // same rounding as upsample_taps
        const float a = __ldg(r0 + x0), b = __ldg(r0 + x1), c = __ldg(r1 + x0), d = __ldg(r1 + x1);
        const float top = a + (b - a) * wx, bot = c + (d - c) * wx;
        v[k] = (top + (bot - top) * wy) * scale;
      }
      if (vec) {
        *reinterpret_cast<float4*>(orow + x4) = make_float4(v[0], v[1], v[2], v[3]);
      } else {
#pragma unroll
        for (int k = 0; k < 4; ++k)
          if (x4 + k < OW) orow[x4 + k] = v[k];
      }
    }
  }
}

// grad_in[i][j] = scale * sum over outputs (y,x) that read input (i,j) of weight * grad_out[y][x]  (gather form)
__global__ void upsample_bwd_kernel(const float* __restrict__ go, float* __restrict__ gi, int planes, int H, int W,
                                    int f, float scale) {
  const int OH = H * f, OW = W * f;
  const long long total = (long long)planes * H * W;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const int j = (int)(idx % W), i = (int)((idx / W) % H);
    const long long pl = idx / ((long long)W * H);
    const float* g = go + pl * OH * OW;
    // candidate output rows: those whose i0 == i (y in [f*i, f*i+f)) or whose i1 == i (i0 == i-1, or i0 == i == H-1 clamp)
    float acc = 0.f;
    const int ylo = max(f * (i - 1), 0), yhi = min(f * (i + 1), OH);
    const int xlo = max(f * (j - 1), 0), xhi = min(f * (j + 1), OW);
    for (int y = ylo; y < yhi; ++y) {
      int y0, y1;
      float wy;
      upsample_taps(y, f, H, y0, y1, wy);
      const float cy = (y0 == i ? 1.f - wy : 0.f) + (y1 == i ? wy : 0.f);
      if (cy == 0.f) continue;
      for (int x = xlo; x < xhi; ++x) {
        int x0, x1;
        float wx;
        upsample_taps(x, f, W, x0, x1, wx);
        const float cx = (x0 == j ? 1.f - wx : 0.f) + (x1 == j ? wx : 0.f);
        acc += cy * cx * __ldg(g + (size_t)y * OW + x);
      }
    }
    gi[idx] = acc * scale;
  }
}

// ---------------------------------------------------------------------------------------------------------
// GridGenerator('warp') and BilinearSampler (network/layer.py:17-18), signature-faithful
// ---------------------------------------------------------------------------------------------------------
__global__ void gridgen_warp_kernel(const float* __restrict__ flow, float* __restrict__ grid, int N, int H, int W) {
  const long long total = (long long)N * H * W;
  const float sx = (float)(W - 1) / 2.f, sy = (float)(H - 1) / 2.f;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const int x = (int)(idx % W), y = (int)((idx / W) % H);
    const long long n = idx / ((long long)W * H);
    const size_t i0 = ((size_t)n * 2) * H * W + (size_t)y * W + x, i1 = i0 + (size_t)H * W;
    grid[i0] = __fdiv_rn(flow[i0] + (float)x, sx) - 1.f;
    grid[i1] = __fdiv_rn(flow[i1] + (float)y, sy) - 1.f;
  }
}

// sampler_taps (the four corners and their weights): sampling.cuh, shared with the backward kernels (image_warp_bwd.cu)
__global__ void bilinear_sampler_kernel(const float* __restrict__ data, const float* __restrict__ grid,
                                        float* __restrict__ out, int N, int C, int H, int W, int OH, int OW) {
  const long long total = (long long)N * OH * OW;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const int x = (int)(idx % OW), y = (int)((idx / OW) % OH);
    const long long n = idx / ((long long)OW * OH);
    const float gx = grid[((size_t)n * 2) * OH * OW + (size_t)y * OW + x];
    const float gy = grid[((size_t)n * 2 + 1) * OH * OW + (size_t)y * OW + x];
    const float xr = (gx + 1.f) * (float)(W - 1) / 2.f, yr = (gy + 1.f) * (float)(H - 1) / 2.f;
    int off[4];
    float wt[4];
    sampler_taps(xr, yr, H, W, off, wt);
    for (int c = 0; c < C; ++c) {
      const float* pl = data + ((size_t)n * C + c) * H * W;
      float v = 0.f;
#pragma unroll
      for (int t = 0; t < 4; ++t)
        if (wt[t] != 0.f) v += __ldg(pl + off[t]) * wt[t];
      out[((size_t)n * C + c) * OH * OW + (size_t)y * OW + x] = v;
    }
  }
}

// K5: c40 = [ sample(im2, pix + Upsample(4)(flow_q)*scale) ; sigmoid(Upsample(4)(mask_q)) - 0.5 ], c30 = [im1 ; 0]
// (network/MaskFlownet.py:308-313).  The grid normalisation of GridGenerator cancels against the sampler's
// de-normalisation, so the source position is pix + displacement directly.  Differentiable: the backward with respect to
// im2, Upsample(4)(flow_q) and Upsample(4)(mask_q) is image_warp_concat_bwd_kernel (image_warp_bwd.cu), and the gradient of
// c30 with respect to im1 is the identity on its first Ci channels.
__global__ void image_warp_concat_kernel(const float* __restrict__ im1, const float* __restrict__ im2,
                                         const float* __restrict__ flow_q, const float* __restrict__ mask_q,
                                         float* __restrict__ c30, float* __restrict__ c40, int N, int Ci, int H, int W,
                                         float scale) {
  const int Hq = H / 4, Wq = W / 4;
  const long long total = (long long)N * H * W;
  const size_t plane = (size_t)H * W;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const int x = (int)(idx % W), y = (int)((idx / W) % H);
    const long long n = idx / ((long long)W * H);
    const float* fq = flow_q + (size_t)n * 2 * Hq * Wq;
    const float fy = upsample_at(fq, Hq, Wq, 4, y, x) * scale;
    const float fx = upsample_at(fq + (size_t)Hq * Wq, Hq, Wq, 4, y, x) * scale;
    const float m = upsample_at(mask_q + (size_t)n * Hq * Wq, Hq, Wq, 4, y, x);
    int off[4];
    float wt[4];
    sampler_taps((float)x + fx, (float)y + fy, H, W, off, wt);
    const size_t pix = (size_t)y * W + x;
    for (int c = 0; c < Ci; ++c) {
      const float* pl = im2 + ((size_t)n * Ci + c) * plane;
      float v = 0.f;
#pragma unroll
      for (int t = 0; t < 4; ++t)
        if (wt[t] != 0.f) v += __ldg(pl + off[t]) * wt[t];
      c40[((size_t)n * (Ci + 1) + c) * plane + pix] = v;
      if (c30) c30[((size_t)n * (Ci + 1) + c) * plane + pix] = __ldg(im1 + ((size_t)n * Ci + c) * plane + pix);
    }
    c40[((size_t)n * (Ci + 1) + Ci) * plane + pix] = sigmoidf_(m) - 0.5f;
    if (c30) c30[((size_t)n * (Ci + 1) + Ci) * plane + pix] = 0.f;
  }
}

// ---------------------------------------------------------------------------------------------------------
// Host dispatch
// ---------------------------------------------------------------------------------------------------------
template <int NT, int FT, int BORDER, bool SHARED>
static void launch_deform_cfg(const float* x, const float* offset, const float* flow_c, const float* mask_c,
                              const float* weight, const float* bias, const float* tradeoff, float* out, float* fup,
                              float* mup, float* conv_out, int N, int C, int H, int W, int F, int up, float fs, float ls,
                              float slope, const int* pix_list, const int* pix_count, cudaStream_t st) {
  const long long total = (long long)N * H * W;
  dim3 grid((unsigned)((total + NT - 1) / NT), (unsigned)((F + FT - 1) / FT));
  deform_fwd_kernel<NT, FT, BORDER, SHARED><<<grid, NT, 0, st>>>(x, offset, flow_c, mask_c, weight, bias, tradeoff, out,
                                                                fup, mup, conv_out, N, C, H, W, F, up, fs, ls, slope,
                                                                pix_list, pix_count);
}

template <int BORDER, bool SHARED>
static int launch_deform(const float* x, const float* offset, const float* flow_c, const float* mask_c,
                         const float* weight, const float* bias, const float* tradeoff, float* out, float* fup,
                         float* mup, float* conv_out, int N, int C, int H, int W, int F, int up, float fs, float ls,
                         float slope, cudaStream_t st, const int* pix_list = nullptr, const int* pix_count = nullptr) {
  // pick (pixels per CTA, output channels per CTA) so that the grid has at least ~3 CTAs per SM; the coarse pyramid
  // levels have only a few thousand pixels
  const long long total = (long long)N * H * W;
  const long long want = 3LL * kNumSMs;
  auto ctas = [&](int nt, int ft) { return ((total + nt - 1) / nt) * ((F + ft - 1) / ft); };
#define MFN_DEFORM_GO(NT_, FT_)                                                                                         \
  launch_deform_cfg<NT_, FT_, BORDER, SHARED>(x, offset, flow_c, mask_c, weight, bias, tradeoff, out, fup, mup, conv_out, \
                                              N, C, H, W, F, up, fs, ls, slope, pix_list, pix_count, st)
  if (F > 32 && ctas(256, 64) >= want) MFN_DEFORM_GO(256, 64);
  else if (ctas(256, 32) >= want) MFN_DEFORM_GO(256, 32);
  else if (F > 32 && ctas(128, 64) >= want) MFN_DEFORM_GO(128, 64);
  else if (ctas(128, 32) >= want) MFN_DEFORM_GO(128, 32);
  else MFN_DEFORM_GO(64, 32);
#undef MFN_DEFORM_GO
  return check_launch(SHARED ? "deform_fwd_kernel<shared-flow>" : "deform_fwd_kernel<per-tap>");
}

}  // namespace mfn

extern "C" int mfn_deformable_conv_forward(const float* data, const float* offset, const float* weight,
                                           const float* bias, float* out, int N, int C, int H, int W, int F,
                                           int kernel_h, int kernel_w, int stride_h, int stride_w, int dilate_h,
                                           int dilate_w, int pad_h, int pad_w, int num_group, int num_deformable_group,
                                           int border_mode, void* stream) {
  using namespace mfn;
  MFN_REQUIRE(data && offset && weight && out, MFN_ERR_INVALID_ARG, "mfn_deformable_conv_forward: null pointer");
  MFN_REQUIRE(N > 0 && C > 0 && H > 0 && W > 0 && F > 0, MFN_ERR_INVALID_ARG,
              "mfn_deformable_conv_forward: non-positive extent");
  MFN_REQUIRE(kernel_h == 3 && kernel_w == 3 && stride_h == 1 && stride_w == 1 && dilate_h == 1 && dilate_w == 1 &&
                  pad_h == 1 && pad_w == 1 && num_group == 1 && num_deformable_group == 1,
              MFN_ERR_UNSUPPORTED,
              "mfn_deformable_conv_forward: only kernel 3x3 / stride 1 / dilate 1 / pad 1 / one group is implemented "
              "(the configuration of network/layer.py:91-95 as instantiated at network/MaskFlownet.py:155-158)");
  MFN_REQUIRE(border_mode == MFN_BORDER_MXNET15 || border_mode == MFN_BORDER_ZERO_CORNER, MFN_ERR_INVALID_ARG,
              "mfn_deformable_conv_forward: unknown border_mode %d", border_mode);
  MFN_REQUIRE((long long)C * H * W < (1LL << 31) && (long long)H * W * 18 < (1LL << 31), MFN_ERR_ALIGNMENT,
              "mfn_deformable_conv_forward: extents overflow kernel indexing");
  cudaStream_t st = as_stream(stream);
  if (border_mode == MFN_BORDER_MXNET15)
    return launch_deform<MFN_BORDER_MXNET15, false>(data, offset, nullptr, nullptr, weight, bias, nullptr, out, nullptr,
                                                    nullptr, nullptr, N, C, H, W, F, 1, 0.f, 1.f, 1.f, st);
  return launch_deform<MFN_BORDER_ZERO_CORNER, false>(data, offset, nullptr, nullptr, weight, bias, nullptr, out,
                                                      nullptr, nullptr, nullptr, N, C, H, W, F, 1, 0.f, 1.f, 1.f, st);
}

extern "C" int mfn_warp_mask_forward(const float* x, const float* flow_coarse, const float* mask_coarse,
                                     const float* weight, const float* bias, const float* tradeoff, float* out,
                                     float* flow_up_out, float* mask_up_out, float* conv_out, int N, int C, int H,
                                     int W, int F, int upsample_factor, float flow_scale, float level_stride,
                                     float leaky_slope, int border_mode, void* stream) {
  using namespace mfn;
  MFN_REQUIRE(x && flow_coarse && weight && out, MFN_ERR_INVALID_ARG, "mfn_warp_mask_forward: null pointer");
  MFN_REQUIRE(N > 0 && C > 0 && H > 0 && W > 0 && F > 0, MFN_ERR_INVALID_ARG,
              "mfn_warp_mask_forward: non-positive extent");
  MFN_REQUIRE(upsample_factor >= 1 && H % upsample_factor == 0 && W % upsample_factor == 0, MFN_ERR_INVALID_ARG,
              "mfn_warp_mask_forward: H and W must be multiples of upsample_factor (H=%d W=%d f=%d)", H, W,
              upsample_factor);
  MFN_REQUIRE(level_stride > 0.f, MFN_ERR_INVALID_ARG, "mfn_warp_mask_forward: level_stride must be positive");
  MFN_REQUIRE(border_mode == MFN_BORDER_MXNET15 || border_mode == MFN_BORDER_ZERO_CORNER, MFN_ERR_INVALID_ARG,
              "mfn_warp_mask_forward: unknown border_mode %d", border_mode);
  MFN_REQUIRE((long long)C * H * W < (1LL << 31) && (long long)F * H * W < (1LL << 31), MFN_ERR_ALIGNMENT,
              "mfn_warp_mask_forward: extents overflow kernel indexing");
  cudaStream_t st = as_stream(stream);
  if (border_mode == MFN_BORDER_MXNET15)
    return launch_deform<MFN_BORDER_MXNET15, true>(x, nullptr, flow_coarse, mask_coarse, weight, bias, tradeoff, out,
                                                   flow_up_out, mask_up_out, conv_out, N, C, H, W, F, upsample_factor,
                                                   flow_scale, level_stride, leaky_slope, st);
  return launch_deform<MFN_BORDER_ZERO_CORNER, true>(x, nullptr, flow_coarse, mask_coarse, weight, bias, tradeoff, out,
                                                     flow_up_out, mask_up_out, conv_out, N, C, H, W, F, upsample_factor,
                                                     flow_scale, level_stride, leaky_slope, st);
}

// ---------------------------------------------------------------------------------------------------------
// K3 through linearity.  All nine taps of the reference's deformable convolution share ONE offset per pixel (the flow is
// `repeat`-ed over the taps, network/MaskFlownet.py:228-232), and bilinear sampling is linear in the image, hence
//     sum_tap W_tap . S(p + tap + f(p))  =  bilinear sample at p + f(p) of  Y = conv3x3(x, W)   (zero padding)
// wherever the nine samples fall strictly inside the image.  The fused warp is therefore
//   (1) Y = plain 3x3 convolution on the tensor cores (conv3x3_wgmma.cu),
//   (2) warp_resample_kernel: per pixel up-sample flow / mask, sample Y, + bias, x sigmoid(mask), + trade-off, LeakyReLU,
//   (3) deform_fwd_kernel over a pixel list: the frame of pixels whose warped centre is within two pixels of the image
//       border, where the operator's border rules (MFN_BORDER_*) are not linear, computed tap by tap as before (the list is
//       built by (2) with one atomic per warp; pixels warped far outside are exact zeros and stay in (2)).
// ---------------------------------------------------------------------------------------------------------
namespace mfn {
__global__ void __launch_bounds__(256)
    warp_resample_kernel(const float* __restrict__ Y, const float* __restrict__ flow_c, const float* __restrict__ mask_c,
                         const float* __restrict__ bias, const float* __restrict__ tradeoff, float* __restrict__ out,
                         float* __restrict__ flow_up_out, float* __restrict__ mask_up_out, int* __restrict__ pix_list,
                         int* __restrict__ pix_count, int N, int H, int W, int F, int up, float flow_scale,
                         float level_stride, float slope) {
  const long long total = (long long)N * H * W;
  const size_t plane = (size_t)H * W;
  const long long span = (long long)gridDim.x * blockDim.x;
  // every warp runs the same number of iterations (the border list is built with warp-wide ballots)
  for (long long base = (long long)blockIdx.x * blockDim.x; base < total; base += span) {
    const long long p = base + threadIdx.x;
    const bool in_range = p < total;
    bool border = false;
    if (in_range) {
    const int xq = (int)(p % W), y = (int)((p / W) % H), n = (int)(p / plane);
    const int Hc = H / up, Wc = W / up;
    const float* fc = flow_c + (size_t)n * 2 * Hc * Wc;
    const float fy = upsample_at(fc, Hc, Wc, up, y, xq);
    const float fx = upsample_at(fc + (size_t)Hc * Wc, Hc, Wc, up, y, xq);
    const float mask_v = mask_c ? upsample_at(mask_c + (size_t)n * Hc * Wc, Hc, Wc, up, y, xq) : 0.f;
    const size_t pix = (size_t)y * W + xq;
    if (flow_up_out) {
      flow_up_out[((size_t)n * 2 + 0) * plane + pix] = fy;
      flow_up_out[((size_t)n * 2 + 1) * plane + pix] = fx;
    }
    if (mask_up_out && mask_c) mask_up_out[(size_t)n * plane + pix] = mask_v;
    const float dy = __fdiv_rn(__fmul_rn(fy, flow_scale), level_stride);
    const float dx = __fdiv_rn(__fmul_rn(fx, flow_scale), level_stride);
    const float h0 = (float)y + dy, w0 = (float)xq + dx;
    const bool inside = warp_interior(h0, w0, H, W);
    border = !inside && !warp_far_outside(h0, w0, H, W);   // served by the tap-by-tap pass
    if (!border) {
      // far outside: all nine taps are zero (w** = 0 below, indices clamped)
      const int i0 = inside ? (int)floorf(h0) : 0, j0 = inside ? (int)floorf(w0) : 0;
      const float lh = h0 - (float)i0, lw = w0 - (float)j0;
      const float z = inside ? 1.f : 0.f;
      const float w00 = z * (1.f - lh) * (1.f - lw), w01 = z * (1.f - lh) * lw, w10 = z * lh * (1.f - lw), w11 = z * lh * lw;
      const float sig = mask_c ? sigmoidf_(mask_v) : 1.f;
      const float* yp = Y + (size_t)n * F * plane + (size_t)i0 * W + j0;
      float* op = out + (size_t)n * F * plane + pix;
      const float* tp = tradeoff ? tradeoff + (size_t)n * F * plane + pix : nullptr;
#pragma unroll 4
      for (int f = 0; f < F; ++f) {
        const float* q = yp + (size_t)f * plane;
        float v = inside ? w00 * __ldg(q) + w01 * __ldg(q + 1) + w10 * __ldg(q + W) + w11 * __ldg(q + W + 1) : 0.f;
        if (bias) v += __ldg(bias + f);
        v *= sig;
        if (tp) v += __ldg(tp + (size_t)f * plane);
        op[(size_t)f * plane] = leaky(v, slope);
      }
    }
    }
    // append the border pixels of this warp to the list: one atomic per warp, lane order kept (neighbours stay together)
    const unsigned ballot = __ballot_sync(0xffffffffu, border);
    if (ballot) {
      const int lane = threadIdx.x & 31;
      int start = 0;
      if (lane == 0) start = atomicAdd(pix_count, __popc(ballot));
      start = __shfl_sync(0xffffffffu, start, 0);
      if (border) pix_list[start + __popc(ballot & ((1u << lane) - 1u))] = (int)p;
    }
  }
}
}  // namespace mfn

extern "C" long long mfn_warp_resample_workspace_bytes(int N, int F, int H, int W) {
  if (N <= 0 || F <= 0 || H <= 0 || W <= 0) return 0;
  const long long list_path = (long long)N * F * H * W * 4 + 16 + (long long)N * H * W * 4;   // Y | border count | border pixel list
  const long long lin_path = mfn::warp_lin_workspace_bytes(N, F, H, W);                          // Yext | Rrow | Rcol | T
  return list_path > lin_path ? list_path : lin_path;
}

extern "C" int mfn_warp_mask_forward_resample(const float* x, const float* flow_coarse, const float* mask_coarse,
                                              const float* weight, const void* packed_weight, const float* bias,
                                              const float* tradeoff, void* workspace, float* out, float* flow_up_out,
                                              float* mask_up_out, int N, int C, int H, int W, int F, int upsample_factor,
                                              float flow_scale, float level_stride, float leaky_slope, int border_mode,
                                              void* stream) {
  using namespace mfn;
  MFN_REQUIRE(x && flow_coarse && weight && packed_weight && workspace && out, MFN_ERR_INVALID_ARG,
              "mfn_warp_mask_forward_resample: null pointer");
  MFN_REQUIRE(aligned(workspace, 16), MFN_ERR_ALIGNMENT, "mfn_warp_mask_forward_resample: workspace must be 16-byte aligned");
  MFN_REQUIRE(N > 0 && C > 0 && H >= 4 && W >= 4 && F > 0 && F <= 256, MFN_ERR_INVALID_ARG,
              "mfn_warp_mask_forward_resample: bad extent (N=%d C=%d H=%d W=%d F=%d)", N, C, H, W, F);
  MFN_REQUIRE(upsample_factor >= 1 && H % upsample_factor == 0 && W % upsample_factor == 0, MFN_ERR_INVALID_ARG,
              "mfn_warp_mask_forward_resample: H and W must be multiples of upsample_factor");
  MFN_REQUIRE(level_stride > 0.f, MFN_ERR_INVALID_ARG, "mfn_warp_mask_forward_resample: level_stride must be positive");
  MFN_REQUIRE(border_mode == MFN_BORDER_MXNET15 || border_mode == MFN_BORDER_ZERO_CORNER, MFN_ERR_INVALID_ARG,
              "mfn_warp_mask_forward_resample: unknown border_mode %d", border_mode);
  MFN_REQUIRE((long long)C * H * W < (1LL << 31) && (long long)F * H * W < (1LL << 31), MFN_ERR_ALIGNMENT,
              "mfn_warp_mask_forward_resample: extents overflow kernel indexing");
  if (tuning().warp_lin) {   // exact evaluation through linearity for every pixel (warp_lin.cu); -1 = extended conv does not fit
    const int rl = launch_warp_lin(x, flow_coarse, mask_coarse, weight, packed_weight, bias, tradeoff, workspace, out, flow_up_out,
                                   mask_up_out, N, C, H, W, F, upsample_factor, flow_scale, level_stride, leaky_slope, border_mode,
                                   as_stream(stream));
    if (rl != -1) return rl;
  }
  float* conv_ws = static_cast<float*>(workspace);
  int* pix_count = reinterpret_cast<int*>(static_cast<unsigned char*>(workspace) + (size_t)N * F * H * W * 4);
  int* pix_list = pix_count + 4;
  // (1) Y = conv3x3(x, W): no bias, no activation
  int rc = mfn_conv3x3_forward_ex(x, 0, packed_weight, nullptr, conv_ws, 0, N, C, H, W, F, 1, 1, MFN_CONV_OUT_NCHW, 1.0f,
                                  stream);
  if (rc) return rc;
  cudaStream_t st = as_stream(stream);
  cudaError_t ce = cudaMemsetAsync(pix_count, 0, 16, st);
  if (ce != cudaSuccess) return fail((int)ce, "mfn_warp_mask_forward_resample: cudaMemsetAsync: %s", cudaGetErrorString(ce));
  // (2) interior (and far-outside) pixels; builds the border list
  const long long total = (long long)N * H * W;
  long long blocks = (total + 255) / 256;
  if (blocks > (long long)kNumSMs * 16) blocks = (long long)kNumSMs * 16;
  warp_resample_kernel<<<(unsigned)blocks, 256, 0, st>>>(conv_ws, flow_coarse, mask_coarse, bias, tradeoff, out, flow_up_out,
                                                        mask_up_out, pix_list, pix_count, N, H, W, F, upsample_factor,
                                                        flow_scale, level_stride, leaky_slope);
  rc = check_launch("warp_resample_kernel");
  if (rc) return rc;
  // (3) the border frame, tap by tap
  if (border_mode == MFN_BORDER_MXNET15)
    return launch_deform<MFN_BORDER_MXNET15, true>(x, nullptr, flow_coarse, mask_coarse, weight, bias, tradeoff, out, nullptr,
                                                   nullptr, nullptr, N, C, H, W, F, upsample_factor, flow_scale,
                                                   level_stride, leaky_slope, st, pix_list, pix_count);
  return launch_deform<MFN_BORDER_ZERO_CORNER, true>(x, nullptr, flow_coarse, mask_coarse, weight, bias, tradeoff, out,
                                                     nullptr, nullptr, nullptr, N, C, H, W, F, upsample_factor, flow_scale,
                                                     level_stride, leaky_slope, st, pix_list, pix_count);
}

extern "C" int mfn_upsample_forward(const float* in, float* out, int planes, int H, int W, int factor, float scale,
                                    void* stream) {
  using namespace mfn;
  MFN_REQUIRE(in && out, MFN_ERR_INVALID_ARG, "mfn_upsample_forward: null pointer");
  MFN_REQUIRE(planes > 0 && H > 0 && W > 0 && factor >= 1, MFN_ERR_INVALID_ARG, "mfn_upsample_forward: bad extent");
  const long long rows = (long long)planes * H * factor;
  const int OW = W * factor, tpb = OW >= 1024 ? 256 : (OW >= 512 ? 128 : 64);
  dim3 grid((unsigned)((OW + 4 * tpb - 1) / (4 * tpb)), (unsigned)(rows < 65535 ? rows : 65535));
  upsample_fwd_kernel<<<grid, tpb, 0, as_stream(stream)>>>(in, out, planes, H, W, factor, scale);
  return check_launch("upsample_fwd_kernel");
}

extern "C" int mfn_upsample_backward(const float* grad_out, float* grad_in, int planes, int H, int W, int factor,
                                     float scale, void* stream) {
  using namespace mfn;
  MFN_REQUIRE(grad_out && grad_in, MFN_ERR_INVALID_ARG, "mfn_upsample_backward: null pointer");
  MFN_REQUIRE(planes > 0 && H > 0 && W > 0 && factor >= 1, MFN_ERR_INVALID_ARG, "mfn_upsample_backward: bad extent");
  const long long total = (long long)planes * H * W;
  upsample_bwd_kernel<<<grid_for(total, 256), 256, 0, as_stream(stream)>>>(grad_out, grad_in, planes, H, W, factor,
                                                                           scale);
  return check_launch("upsample_bwd_kernel");
}

extern "C" int mfn_grid_generator_warp_forward(const float* flow_xy, float* grid, int N, int H, int W, void* stream) {
  using namespace mfn;
  MFN_REQUIRE(flow_xy && grid, MFN_ERR_INVALID_ARG, "mfn_grid_generator_warp_forward: null pointer");
  MFN_REQUIRE(N > 0 && H > 1 && W > 1, MFN_ERR_INVALID_ARG, "mfn_grid_generator_warp_forward: need H, W > 1");
  gridgen_warp_kernel<<<grid_for((long long)N * H * W, 256), 256, 0, as_stream(stream)>>>(flow_xy, grid, N, H, W);
  return check_launch("gridgen_warp_kernel");
}

extern "C" int mfn_bilinear_sampler_forward(const float* data, const float* grid, float* out, int N, int C, int H,
                                            int W, int OH, int OW, void* stream) {
  using namespace mfn;
  MFN_REQUIRE(data && grid && out, MFN_ERR_INVALID_ARG, "mfn_bilinear_sampler_forward: null pointer");
  MFN_REQUIRE(N > 0 && C > 0 && H > 0 && W > 0 && OH > 0 && OW > 0, MFN_ERR_INVALID_ARG,
              "mfn_bilinear_sampler_forward: bad extent");
  bilinear_sampler_kernel<<<grid_for((long long)N * OH * OW, 256), 256, 0, as_stream(stream)>>>(data, grid, out, N, C,
                                                                                              H, W, OH, OW);
  return check_launch("bilinear_sampler_kernel");
}

extern "C" int mfn_image_warp_concat_forward(const float* im1, const float* im2, const float* flow_q,
                                             const float* mask_q, float* c30, float* c40, int N, int Ci, int H, int W,
                                             float flow_scale, void* stream) {
  using namespace mfn;
  MFN_REQUIRE(im2 && flow_q && mask_q && c40, MFN_ERR_INVALID_ARG, "mfn_image_warp_concat_forward: null pointer");
  MFN_REQUIRE(!c30 || im1, MFN_ERR_INVALID_ARG, "mfn_image_warp_concat_forward: c30 requested without im1");
  MFN_REQUIRE(N > 0 && Ci > 0 && H > 0 && W > 0 && H % 4 == 0 && W % 4 == 0, MFN_ERR_INVALID_ARG,
              "mfn_image_warp_concat_forward: H and W must be positive multiples of 4");
  image_warp_concat_kernel<<<grid_for((long long)N * H * W, 256), 256, 0, as_stream(stream)>>>(
      im1, im2, flow_q, mask_q, c30, c40, N, Ci, H, W, flow_scale);
  return check_launch("image_warp_concat_kernel");
}
