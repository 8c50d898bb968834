// loss.cu -- MultiscaleEpe('upsampling') of the reference, fused (SURVEY.md section 8f, row N2: "MultiscaleEpe as one fused
// kernel"); reference: network/MaskFlownet.py:563-611 (EpeLossWithMask, MultiscaleEpe), built in network/pipeline.py:39-45 with
// scales (64, 32, 16, 8, 4) and weights (.005, .01, .02, .08, .32), applied in pipeline.py:81-83, 107.
//
//   loss[n] = sum_s w_s * ( sum_hw e_s(y,x) * mask(y,x) ) / sum_hw mask(y,x),
//   e_s = sqrt( sum_c (Upsample(s)(pred_s)_c - flow_c)^2 + eps )            (q given:  (sum_c |.| + eps)^q )
//
// The reference materialises Upsample(s)(pred_s) at full resolution for each of the five scales (a transposed convolution
// with a (2s-1)^2 kernel), then ~8 element-wise / reduction operators per scale, and the mirror image of all of it in the
// backward pass.  Here:
//   forward   one pass over the full-resolution pixels: flow and mask are read ONCE, the five up-sampled predictions are
//             evaluated on the fly from the (tiny, cache-resident) coarse tensors, per-block partial sums, a finishing launch
//             (fixed summation order: bit-reproducible);
//   backward  one launch, gather form, one warp per coarse prediction pixel: it walks the <= (2s)^2 full-resolution pixels
//             that read that coarse pixel, recomputes e_s there and reduces  w_s * mask * (up - flow) / e_s * tap weight
//             (no full-resolution gradient tensor is ever written; no atomics).
// Algorithmic bytes: forward 4*N*H*W*3 (flow + mask) + the coarse tensors; backward the same per scale from L2.
#ifdef MFN_HOST_EMULATION
#include "cuda_shim.h"
#include "device_caps.h"
#include "sampling.cuh"
#else
#include "common.cuh"
#endif

namespace mfn {
namespace epe {

constexpr int MAX_SCALES = 8;
#ifdef MFN_HOST_EMULATION
constexpr int LANES = 1;     // the shim runs one lane per "warp" (its shuffle returns the caller's own value)
#else
constexpr int LANES = 32;
#endif

struct Args {
  const float* pred[MAX_SCALES];    // (N, 2, H / s, W / s)
  float* gpred[MAX_SCALES];         // backward only
  int scale[MAX_SCALES];
  float weight[MAX_SCALES];
  long long first_warp[MAX_SCALES + 1];   // backward: prefix sums of N * (H / s) * (W / s)
  int num;
};

// both channels of Upsample(f)(pred)[n] at (y, x); same interpolation order as upsample_at (sampling.cuh)
__device__ __forceinline__ void upsample2_at(const float* __restrict__ p, int Hc, int Wc, int f, int y, int x, float& u0,
                                             float& u1) {
  int y0, y1, x0, x1;
  float wy, wx;
  upsample_taps(y, f, Hc, y0, y1, wy);
  upsample_taps(x, f, Wc, x0, x1, wx);
  const size_t cp = (size_t)Hc * Wc;
  const int o00 = y0 * Wc + x0, o01 = y0 * Wc + x1, o10 = y1 * Wc + x0, o11 = y1 * Wc + x1;
  {
    const float a = __ldg(p + o00), b = __ldg(p + o01), c = __ldg(p + o10), d = __ldg(p + o11);
    const float top = a + (b - a) * wx, bot = c + (d - c) * wx;
    u0 = top + (bot - top) * wy;
  }
  {
    const float a = __ldg(p + cp + o00), b = __ldg(p + cp + o01), c = __ldg(p + cp + o10), d = __ldg(p + cp + o11);
    const float top = a + (b - a) * wx, bot = c + (d - c) * wx;
    u1 = top + (bot - top) * wy;
  }
}

// e and d e / d up_c for one pixel and scale (MaskFlownet.py:577-580)
__device__ __forceinline__ float epe_value(float d0, float d1, float eps, float q) {
  if (q >= 0.f) return powf(fabsf(d0) + fabsf(d1) + eps, q);
  return sqrtf(d0 * d0 + d1 * d1 + eps);
}
__device__ __forceinline__ void epe_grad(float d0, float d1, float eps, float q, float& g0, float& g1) {
  if (q >= 0.f) {
    const float k = q * powf(fabsf(d0) + fabsf(d1) + eps, q - 1.f);
    g0 = d0 > 0.f ? k : (d0 < 0.f ? -k : 0.f);
    g1 = d1 > 0.f ? k : (d1 < 0.f ? -k : 0.f);
  } else {
    const float r = 1.f / sqrtf(d0 * d0 + d1 * d1 + eps);
    g0 = d0 * r;
    g1 = d1 * r;
  }
}

// sum over the block of two values; valid in thread 0.  blockDim.x a multiple of LANES, <= 1024.
__device__ __forceinline__ void block_sum2(float& a, float& b) {
  __shared__ float red[2][32];
  for (int o = LANES / 2; o > 0; o >>= 1) {
    a += __shfl_xor_sync(0xffffffffu, a, o);
    b += __shfl_xor_sync(0xffffffffu, b, o);
  }
  const int lane = threadIdx.x % LANES, warp = threadIdx.x / LANES, nwarps = (blockDim.x + LANES - 1) / LANES;
  if (lane == 0) {
    red[0][warp] = a;
    red[1][warp] = b;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    a = b = 0.f;
    for (int w = 0; w < nwarps; ++w) {      // fixed order
      a += red[0][w];
      b += red[1][w];
    }
  }
}

// grid (blocks per sample, N): partial[n][block] = (sum_hw mask * sum_s w_s e_s, sum_hw mask) over the block's pixels
__global__ void __launch_bounds__(256)
    epe_forward_kernel(const float* __restrict__ flow, const float* __restrict__ mask, Args A, float eps, float q,
                       float* __restrict__ partial, int H, int W) {
  const int n = blockIdx.y, HW = H * W;
  const float* f0 = flow + (size_t)n * 2 * HW;
  const float* m = mask + (size_t)n * HW;
  float num = 0.f, den = 0.f;
  for (int pix = blockIdx.x * blockDim.x + threadIdx.x; pix < HW; pix += gridDim.x * blockDim.x) {
    const int y = pix / W, x = pix - y * W;
    const float fy = __ldg(f0 + pix), fx = __ldg(f0 + HW + pix), mv = __ldg(m + pix);
    float e = 0.f;
    for (int s = 0; s < A.num; ++s) {
      const int f = A.scale[s], Hc = H / f, Wc = W / f;
      float u0, u1;
      upsample2_at(A.pred[s] + (size_t)n * 2 * Hc * Wc, Hc, Wc, f, y, x, u0, u1);
      e += A.weight[s] * epe_value(u0 - fy, u1 - fx, eps, q);
    }
    num += e * mv;
    den += mv;
  }
  block_sum2(num, den);
  if (threadIdx.x == 0) {
    partial[((size_t)n * gridDim.x + blockIdx.x) * 2 + 0] = num;
    partial[((size_t)n * gridDim.x + blockIdx.x) * 2 + 1] = den;
  }
}

__global__ void epe_finish_kernel(const float* __restrict__ partial, float* __restrict__ loss, float* __restrict__ mask_sum,
                                  int N, int blocks) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= N) return;
  float num = 0.f, den = 0.f;
  for (int b = 0; b < blocks; ++b) {
    num += partial[((size_t)n * blocks + b) * 2 + 0];
    den += partial[((size_t)n * blocks + b) * 2 + 1];
  }
  loss[n] = num / den;            // an all-zero mask divides by zero, as the reference does (MaskFlownet.py:582)
  mask_sum[n] = den;
}

// one warp per coarse prediction pixel (scale s, sample n, row i, column j): both channels' gradients
__global__ void __launch_bounds__(256)
    epe_backward_kernel(const float* __restrict__ flow, const float* __restrict__ mask, Args A, float eps, float q,
                        const float* __restrict__ grad_loss, const float* __restrict__ mask_sum, int N, int H, int W) {
  const int lane = threadIdx.x % LANES;
  const long long warps_per_grid = (long long)gridDim.x * (blockDim.x / LANES);
  const int HW = H * W;
  for (long long w = (long long)blockIdx.x * (blockDim.x / LANES) + threadIdx.x / LANES; w < A.first_warp[A.num];
       w += warps_per_grid) {
    int s = 0;
    while (s + 1 < A.num && w >= A.first_warp[s + 1]) ++s;
    const int f = A.scale[s], Hc = H / f, Wc = W / f;
    const long long r = w - A.first_warp[s];
    const int j = (int)(r % Wc), i = (int)((r / Wc) % Hc), n = (int)(r / ((long long)Wc * Hc));
    const float* p = A.pred[s] + (size_t)n * 2 * Hc * Wc;
    const float* f0 = flow + (size_t)n * 2 * HW;
    const float* m = mask + (size_t)n * HW;
    // full-resolution pixels whose taps include (i, j): rows f*(i-1) .. f*(i+1)-1 (and the clamped last row / column)
    const int ylo = max(f * (i - 1), 0), yhi = min(f * (i + 1), H), xlo = max(f * (j - 1), 0), xhi = min(f * (j + 1), W);
    const int nx = xhi - xlo, cnt = (yhi - ylo) * nx;
    float a0 = 0.f, a1 = 0.f;
    for (int k = lane; k < cnt; k += LANES) {
      const int y = ylo + k / nx, x = xlo + k % nx;
      int y0, y1, x0, x1;
      float wy, wx;
      upsample_taps(y, f, Hc, y0, y1, wy);
      upsample_taps(x, f, Wc, x0, x1, wx);
      const float cy = (y0 == i ? 1.f - wy : 0.f) + (y1 == i ? wy : 0.f);
      const float cx = (x0 == j ? 1.f - wx : 0.f) + (x1 == j ? wx : 0.f);
      const float mv = __ldg(m + y * W + x), coef = cy * cx * mv;
      if (coef == 0.f) continue;
      float u0, u1, g0, g1;
      upsample2_at(p, Hc, Wc, f, y, x, u0, u1);
      epe_grad(u0 - __ldg(f0 + y * W + x), u1 - __ldg(f0 + HW + y * W + x), eps, q, g0, g1);
      a0 += coef * g0;
      a1 += coef * g1;
    }
    for (int o = LANES / 2; o > 0; o >>= 1) {
      a0 += __shfl_xor_sync(0xffffffffu, a0, o);
      a1 += __shfl_xor_sync(0xffffffffu, a1, o);
    }
    if (lane == 0) {
      const float k = A.weight[s] * __ldg(grad_loss + n) / __ldg(mask_sum + n);
      float* g = A.gpred[s] + (size_t)n * 2 * Hc * Wc + (size_t)i * Wc + j;
      g[0] = a0 * k;
      g[(size_t)Hc * Wc] = a1 * k;
    }
  }
}

constexpr int FWD_BLOCKS = 64;   // per sample

}  // namespace epe
}  // namespace mfn

#ifndef MFN_HOST_EMULATION
namespace {
int fill_args(mfn::epe::Args& A, const float* const* preds, float* const* gpreds, const int* scales, const float* weights,
              int num_scales, int N, int H, int W, const char* who) {
  using namespace mfn;
  MFN_REQUIRE(preds && scales && weights, MFN_ERR_INVALID_ARG, "%s: null pointer", who);
  MFN_REQUIRE(num_scales >= 1 && num_scales <= epe::MAX_SCALES, MFN_ERR_INVALID_ARG, "%s: 1 <= num_scales <= %d", who,
              epe::MAX_SCALES);
  MFN_REQUIRE(N > 0 && H > 0 && W > 0 && (long long)H * W * 2 < (1LL << 31), MFN_ERR_INVALID_ARG, "%s: bad extent", who);
  A.num = num_scales;
  A.first_warp[0] = 0;
  for (int s = 0; s < num_scales; ++s) {
    MFN_REQUIRE(preds[s] && (!gpreds || gpreds[s]), MFN_ERR_INVALID_ARG, "%s: null prediction pointer %d", who, s);
    MFN_REQUIRE(scales[s] >= 1 && H % scales[s] == 0 && W % scales[s] == 0, MFN_ERR_INVALID_ARG,
                "%s: scale %d does not divide %dx%d (Upsample(s)(pred) must have the label's size)", who, scales[s], H, W);
    A.pred[s] = preds[s];
    A.gpred[s] = gpreds ? gpreds[s] : nullptr;
    A.scale[s] = scales[s];
    A.weight[s] = weights[s];
    A.first_warp[s + 1] = A.first_warp[s] + (long long)N * (H / scales[s]) * (W / scales[s]);
  }
  return MFN_OK;
}
}  // namespace

extern "C" long long mfn_multiscale_epe_workspace_bytes(int N) {
  return N > 0 ? (long long)N * mfn::epe::FWD_BLOCKS * 2 * (long long)sizeof(float) : 0;
}

extern "C" int mfn_multiscale_epe_forward(const float* flow, const float* mask, const float* const* preds, const int* scales,
                                          const float* weights, int num_scales, float eps, float q, float* loss,
                                          float* mask_sum, void* workspace, long long workspace_bytes, int N, int H, int W,
                                          void* stream) {
  using namespace mfn;
  MFN_REQUIRE(flow && mask && loss && mask_sum && workspace, MFN_ERR_INVALID_ARG, "mfn_multiscale_epe_forward: null pointer");
  MFN_REQUIRE(N <= 65535, MFN_ERR_INVALID_ARG, "mfn_multiscale_epe_forward: N > 65535");
  epe::Args A;
  int rc = fill_args(A, preds, nullptr, scales, weights, num_scales, N, H, W, "mfn_multiscale_epe_forward");
  if (rc) return rc;
  MFN_REQUIRE(workspace_bytes >= mfn_multiscale_epe_workspace_bytes(N), MFN_ERR_INVALID_ARG,
              "mfn_multiscale_epe_forward: workspace smaller than mfn_multiscale_epe_workspace_bytes(N)");
  cudaStream_t st = as_stream(stream);
  float* partial = static_cast<float*>(workspace);
  epe::epe_forward_kernel<<<dim3(epe::FWD_BLOCKS, N), 256, 0, st>>>(flow, mask, A, eps, q, partial, H, W);
  rc = check_launch("epe_forward_kernel");
  if (rc) return rc;
  epe::epe_finish_kernel<<<(N + 127) / 128, 128, 0, st>>>(partial, loss, mask_sum, N, epe::FWD_BLOCKS);
  return check_launch("epe_finish_kernel");
}

extern "C" int mfn_multiscale_epe_backward(const float* flow, const float* mask, const float* const* preds, const int* scales,
                                           const float* weights, int num_scales, float eps, float q, const float* grad_loss,
                                           const float* mask_sum, float* const* grad_preds, int N, int H, int W,
                                           void* stream) {
  using namespace mfn;
  MFN_REQUIRE(flow && mask && grad_loss && mask_sum && grad_preds, MFN_ERR_INVALID_ARG,
              "mfn_multiscale_epe_backward: null pointer");
  epe::Args A;
  int rc = fill_args(A, preds, grad_preds, scales, weights, num_scales, N, H, W, "mfn_multiscale_epe_backward");
  if (rc) return rc;
  const long long warps = A.first_warp[A.num];
  long long blocks = (warps + 7) / 8;     // 8 warps per block
  if (blocks > (long long)kNumSMs * 64) blocks = (long long)kNumSMs * 64;
  epe::epe_backward_kernel<<<(unsigned)blocks, 256, 0, as_stream(stream)>>>(flow, mask, A, eps, q, grad_loss, mask_sum, N, H, W);
  return check_launch("epe_backward_kernel");
}
#endif  // !MFN_HOST_EMULATION
