// unsup_loss.cu -- the photometric and smoothness losses of unsupervised fine-tuning on unlabelled frame pairs (the
// recipe of UnFlow, Meister, Hur and Roth, AAAI 2018): a census-transform distance between image 1 and image 2 warped by
// the flow, masked by the forward-backward occlusion check, and a second-order, edge-aware smoothness of the flow.
//
//   census    img1, img2w (N,3,H,W) in [0,1], occ (N,H,W) uint8  ->  loss (N), vsum (N), coef (N,H,W)
//     I = 255 (0.2989 R + 0.5870 G + 0.1140 B); on interior pixels p (3 <= x <= W-4, 3 <= y <= H-4), over the 48 offsets
//     o of the 7x7 window without its centre:  t(I,p,o) = D / sqrt(0.81 + D^2), D = I(p+o) - I(p);  s = t(I1) - t(I2w);
//     d(p) = sum_o s^2 / (0.1 + s^2);  rho(d) = (d^2 + 1e-6)^0.45;  v = 1 - occ on interior pixels, 0 elsewhere;
//     loss[n] = sum_p v rho(d) / max(sum_p v, 1),  vsum[n] = sum_p v,  coef = v rho'(d) (kept for the backward).
//     forward  one CTA per 32 x 8 output tile stages both grey planes with a 3-pixel halo in shared memory (RGB -> grey
//              on load); per-CTA partial sums go to the workspace and one finishing launch adds them in a fixed order.
//     backward a gather, every element of g_img2w written once.  With h(p,o) = d d(p) / d D2 =
//              -0.2 s / (0.1 + s^2)^2 * 0.81 / (0.81 + D2^2)^(3/2), the grey gradient at q is
//                sum_o coef(q-o) h(q-o,o) - coef(q) sum_o h(q,o)  =  -sum_o (coef(q+o) + coef(q)) h(q,o),
//              because h(q+o,-o) = -h(q,o) exactly in fp32 as well (t is odd and D(q+o,-o) = -D(q,o) is exact): one h
//              per offset and pixel, from the values at q and q+o, so a 3-pixel halo of coef and both grey planes is
//              enough.  Times g_loss[n] / max(vsum[n], 1), then 255 (0.2989, 0.5870, 0.1140) for the RGB gradient.
//
//   smoothness  flow (N,2,H,W), img (N,3,H,W)  ->  loss (N)
//     d2x F_c = F_c(x-1) - 2 F_c(x) + F_c(x+1) (1 <= x <= W-2), wx = exp(-10 (1/3) sum_k |img_k(x+1) - img_k(x-1)| / 2),
//     the same in y;  loss[n] = sum_{c,p} wx |d2x F_c| / (2 H (W-2)) + sum_{c,p} wy |d2y F_c| / (2 (H-2) W).
//     forward  one thread per pixel, per-CTA partial sums of the x and y terms, the same finishing launch.
//     backward a 3-tap gather per direction; d|z|/dz = sign(z), 0 at 0.
//
// No atomics anywhere: every result is bit-reproducible.  Shapes below 7 (census) or 3 (smoothness) in a dimension have
// no interior pixels and give a loss of 0.  The file also builds for the host (MFN_HOST_EMULATION:
// tests/host_emu/unsup_loss_emu.cpp), one thread per block: the loops over a tile's pixels and the tree reductions take
// any power-of-two blockDim.x up to their tile size.
#ifdef MFN_HOST_EMULATION
#include "cuda_shim.h"
#else
#include <math.h>

#include "common.cuh"
#endif

namespace mfn {
namespace unsup {

constexpr int R = 3;                              // census window radius
constexpr int TW = 32, TH = 8, NT = TW * TH;      // census output tile (one CTA) and its threads
constexpr int SW = TW + 2 * R, SH = TH + 2 * R;   // staged tile with halo
constexpr int SNT = 256;                          // smoothness: pixels (threads) per CTA
constexpr int FNT = 256;                          // finishing launch: threads per sample

__device__ __forceinline__ float grey(const float* __restrict__ img, size_t plane, size_t i) {
  return 255.f * (0.2989f * __ldg(img + i) + 0.5870f * __ldg(img + plane + i) + 0.1140f * __ldg(img + 2 * plane + i));
}

__device__ __forceinline__ float census_t(float d) { return d / sqrtf(0.81f + d * d); }

// d(p) from grey planes g1, g2 (row stride ld) at the centre pixel they point to; every read is within R of it.
__device__ __forceinline__ float census_distance(const float* g1, const float* g2, int ld) {
  const float c1 = g1[0], c2 = g2[0];
  float d = 0.f;
  for (int dy = -R; dy <= R; ++dy)
    for (int dx = -R; dx <= R; ++dx) {
      if (dy == 0 && dx == 0) continue;
      const int o = dy * ld + dx;
      const float s = census_t(g1[o] - c1) - census_t(g2[o] - c2);
      d += s * s / (0.1f + s * s);
    }
  return d;
}

__device__ __forceinline__ bool census_interior(int x, int y, int H, int W) {
  return x >= R && x < W - R && y >= R && y < H - R;
}

// the block's sums of a and b in red[.][0] (fixed tree order); blockDim.x a power of two <= NTH
template <int NTH>
__device__ __forceinline__ void block_sum2(float a, float b, float (*red)[NTH]) {
  const int t = threadIdx.x;
  red[0][t] = a;
  red[1][t] = b;
  __syncthreads();
  for (int s = blockDim.x / 2; s > 0; s >>= 1) {
    if (t < s) {
      red[0][t] += red[0][t + s];
      red[1][t] += red[1][t + s];
    }
    __syncthreads();
  }
}

// both grey planes of sample n over the tile at (x0 - R, y0 - R), SH x SW, zero outside the image
__device__ __forceinline__ void stage_grey(const float* __restrict__ i1, const float* __restrict__ i2, float* g1, float* g2,
                                           int x0, int y0, int H, int W) {
  const size_t plane = (size_t)H * W;
  for (int k = threadIdx.x; k < SH * SW; k += blockDim.x) {
    const int ty = k / SW, tx = k - ty * SW, y = y0 - R + ty, x = x0 - R + tx;
    const bool in = y >= 0 && y < H && x >= 0 && x < W;
    const size_t i = (size_t)y * W + x;
    g1[k] = in ? grey(i1, plane, i) : 0.f;
    g2[k] = in ? grey(i2, plane, i) : 0.f;
  }
}

// grid (ceil(W / TW), ceil(H / TH), N): coef of the tile's pixels, partial[(n, tile)] = (sum v rho(d), sum v)
__global__ void __launch_bounds__(NT)
    census_forward_kernel(const float* __restrict__ img1, const float* __restrict__ img2w,
                          const unsigned char* __restrict__ occ, float* __restrict__ coef, float* __restrict__ partial,
                          int H, int W) {
  __shared__ float g1[SH * SW], g2[SH * SW];
  __shared__ float red[2][NT];
  const int n = blockIdx.z, x0 = blockIdx.x * TW, y0 = blockIdx.y * TH;
  const size_t plane = (size_t)H * W;
  stage_grey(img1 + (size_t)n * 3 * plane, img2w + (size_t)n * 3 * plane, g1, g2, x0, y0, H, W);
  __syncthreads();
  float num = 0.f, den = 0.f;
  for (int k = threadIdx.x; k < NT; k += blockDim.x) {
    const int ty = k / TW, tx = k - ty * TW, y = y0 + ty, x = x0 + tx;
    if (y >= H || x >= W) continue;
    const size_t i = (size_t)n * plane + (size_t)y * W + x;
    float c = 0.f;
    if (census_interior(x, y, H, W) && __ldg(occ + i) == 0) {
      const int s = (ty + R) * SW + tx + R;
      const float d = census_distance(g1 + s, g2 + s, SW);
      const float q = d * d + 1e-6f;
      num += powf(q, 0.45f);
      den += 1.f;
      c = 0.9f * d * powf(q, -0.55f);
    }
    coef[i] = c;
  }
  block_sum2<NT>(num, den, red);
  if (threadIdx.x == 0) {
    const size_t t = ((size_t)n * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x;
    partial[2 * t] = red[0][0];
    partial[2 * t + 1] = red[1][0];
  }
}

// grid (N): adds the sample's `parts` partial pairs in a fixed order.  census: loss = a / max(b, 1), vsum = b;
// smoothness (vsum null): loss = a / (2 H (W-2)) + b / (2 (H-2) W), a term without pixels counting 0.
__global__ void __launch_bounds__(FNT)
    finish_kernel(const float* __restrict__ partial, int parts, float* __restrict__ loss, float* __restrict__ vsum, int H,
                  int W) {
  __shared__ float red[2][FNT];
  const int n = blockIdx.x;
  float a = 0.f, b = 0.f;
  for (int t = threadIdx.x; t < parts; t += blockDim.x) {
    a += partial[2 * ((size_t)n * parts + t)];
    b += partial[2 * ((size_t)n * parts + t) + 1];
  }
  block_sum2<FNT>(a, b, red);
  if (threadIdx.x != 0) return;
  a = red[0][0];
  b = red[1][0];
  if (vsum) {
    loss[n] = a / fmaxf(b, 1.f);
    vsum[n] = b;
  } else {
    loss[n] = (W > 2 ? a / (2.f * (float)H * (float)(W - 2)) : 0.f) + (H > 2 ? b / (2.f * (float)(H - 2) * (float)W) : 0.f);
  }
}

// grid (ceil(W / TW), ceil(H / TH), N): g_img2w of the tile's pixels
__global__ void __launch_bounds__(NT)
    census_backward_kernel(const float* __restrict__ img1, const float* __restrict__ img2w, const float* __restrict__ coef,
                           const float* __restrict__ vsum, const float* __restrict__ g_loss, float* __restrict__ g_img2w,
                           int H, int W) {
  __shared__ float g1[SH * SW], g2[SH * SW], cf[SH * SW];
  const int n = blockIdx.z, x0 = blockIdx.x * TW, y0 = blockIdx.y * TH;
  const size_t plane = (size_t)H * W;
  stage_grey(img1 + (size_t)n * 3 * plane, img2w + (size_t)n * 3 * plane, g1, g2, x0, y0, H, W);
  const float* cn = coef + (size_t)n * plane;
  for (int k = threadIdx.x; k < SH * SW; k += blockDim.x) {
    const int ty = k / SW, tx = k - ty * SW, y = y0 - R + ty, x = x0 - R + tx;
    cf[k] = (y >= 0 && y < H && x >= 0 && x < W) ? __ldg(cn + (size_t)y * W + x) : 0.f;
  }
  __syncthreads();
  const float scale = 255.f * (__ldg(g_loss + n) / fmaxf(__ldg(vsum + n), 1.f));
  float* go = g_img2w + (size_t)n * 3 * plane;
  for (int k = threadIdx.x; k < NT; k += blockDim.x) {
    const int ty = k / TW, tx = k - ty * TW, y = y0 + ty, x = x0 + tx;
    if (y >= H || x >= W) continue;
    const int s = (ty + R) * SW + tx + R;
    const float c1 = g1[s], c2 = g2[s], cq = cf[s];
    float acc = 0.f;
    for (int dy = -R; dy <= R; ++dy)
      for (int dx = -R; dx <= R; ++dx) {
        if (dy == 0 && dx == 0) continue;
        const int o = s + dy * SW + dx;
        const float d2 = g2[o] - c2;
        const float r2 = 0.81f + d2 * d2, sq = sqrtf(r2);
        const float sv = census_t(g1[o] - c1) - d2 / sq;   // d2 / sq is census_t(d2), operation for operation
        const float q = 0.1f + sv * sv;
        const float h = -0.2f * sv / (q * q) * (0.81f / (r2 * sq));
        acc += (cf[o] + cq) * h;
      }
    const float g = -acc * scale;
    const size_t i = (size_t)y * W + x;
    go[i] = g * 0.2989f;
    go[plane + i] = g * 0.5870f;
    go[2 * plane + i] = g * 0.1140f;
  }
}

// exp(-10 (1/3) sum_k |img_k(j) - img_k(i)| / 2) for the pixels i and j of one sample's image
__device__ __forceinline__ float edge_weight(const float* __restrict__ img, size_t plane, size_t i, size_t j) {
  const float e = fabsf(__ldg(img + j) - __ldg(img + i)) + fabsf(__ldg(img + plane + j) - __ldg(img + plane + i)) +
                  fabsf(__ldg(img + 2 * plane + j) - __ldg(img + 2 * plane + i));
  return expf(-10.f * (0.5f * (e / 3.f)));
}

__device__ __forceinline__ float second_diff(const float* __restrict__ f, size_t i, size_t step) {
  return __ldg(f + i - step) - 2.f * __ldg(f + i) + __ldg(f + i + step);
}

// grid (ceil(H W / SNT), N): partial[(n, block)] = (sum wx |d2x F|, sum wy |d2y F|) over the block's pixels
__global__ void __launch_bounds__(SNT)
    smoothness_forward_kernel(const float* __restrict__ flow, const float* __restrict__ img, float* __restrict__ partial,
                              int H, int W) {
  __shared__ float red[2][SNT];
  const int n = blockIdx.y;
  const size_t plane = (size_t)H * W;
  const float* f = flow + (size_t)n * 2 * plane;
  const float* im = img + (size_t)n * 3 * plane;
  float sx = 0.f, sy = 0.f;
  for (int k = threadIdx.x; k < SNT; k += blockDim.x) {
    const long long p = (long long)blockIdx.x * SNT + k;
    if (p >= (long long)plane) continue;
    const int y = (int)(p / W), x = (int)(p - (long long)y * W);
    if (x >= 1 && x <= W - 2) {
      const float w = edge_weight(im, plane, p - 1, p + 1);
      sx += w * (fabsf(second_diff(f, p, 1)) + fabsf(second_diff(f + plane, p, 1)));
    }
    if (y >= 1 && y <= H - 2) {
      const float w = edge_weight(im, plane, p - W, p + W);
      sy += w * (fabsf(second_diff(f, p, W)) + fabsf(second_diff(f + plane, p, W)));
    }
  }
  block_sum2<SNT>(sx, sy, red);
  if (threadIdx.x == 0) {
    const size_t t = (size_t)n * gridDim.x + blockIdx.x;
    partial[2 * t] = red[0][0];
    partial[2 * t + 1] = red[1][0];
  }
}

__device__ __forceinline__ float sign_of(float z) { return z > 0.f ? 1.f : (z < 0.f ? -1.f : 0.f); }

// grid (ceil(H W / SNT), N): g_flow at the block's pixels, both channels.  The pixel q is the centre (weight -2) of its
// own stencil and a side tap (weight 1) of its neighbours' stencils, in each direction.
__global__ void __launch_bounds__(SNT)
    smoothness_backward_kernel(const float* __restrict__ flow, const float* __restrict__ img,
                               const float* __restrict__ g_loss, float* __restrict__ g_flow, int H, int W) {
  const int n = blockIdx.y;
  const size_t plane = (size_t)H * W;
  const float* f = flow + (size_t)n * 2 * plane;
  const float* im = img + (size_t)n * 3 * plane;
  const float g = __ldg(g_loss + n);
  const float kx = W > 2 ? g / (2.f * (float)H * (float)(W - 2)) : 0.f;
  const float ky = H > 2 ? g / (2.f * (float)(H - 2) * (float)W) : 0.f;
  for (int k = threadIdx.x; k < SNT; k += blockDim.x) {
    const long long p = (long long)blockIdx.x * SNT + k;
    if (p >= (long long)plane) continue;
    const int y = (int)(p / W), x = (int)(p - (long long)y * W);
    float ax[2] = {0.f, 0.f}, ay[2] = {0.f, 0.f};
    for (int j = -1; j <= 1; ++j) {
      const float tap = j == 0 ? -2.f : 1.f;
      const int xc = x + j, yc = y + j;
      if (xc >= 1 && xc <= W - 2) {
        const size_t c = p + j;
        const float w = tap * edge_weight(im, plane, c - 1, c + 1);
        for (int ch = 0; ch < 2; ++ch) ax[ch] += w * sign_of(second_diff(f + ch * plane, c, 1));
      }
      if (yc >= 1 && yc <= H - 2) {
        const size_t c = p + (long long)j * W;
        const float w = tap * edge_weight(im, plane, c - W, c + W);
        for (int ch = 0; ch < 2; ++ch) ay[ch] += w * sign_of(second_diff(f + ch * plane, c, W));
      }
    }
    float* go = g_flow + (size_t)n * 2 * plane;
    go[p] = ax[0] * kx + ay[0] * ky;
    go[plane + p] = ax[1] * kx + ay[1] * ky;
  }
}

}  // namespace unsup
}  // namespace mfn

#ifndef MFN_HOST_EMULATION
namespace {
// the checks every entry point shares: positive extents, 4-byte aligned float pointers, int pixel indices, grid limits
int check_extents(int N, int H, int W, const char* who) {
  using namespace mfn;
  MFN_REQUIRE(N > 0 && H > 0 && W > 0, MFN_ERR_INVALID_ARG, "%s: non-positive extent", who);
  MFN_REQUIRE((long long)H * W * 3 < (1LL << 31) && N <= 65535, MFN_ERR_INVALID_ARG,
              "%s: extents overflow kernel indexing (3*H*W < 2^31, N <= 65535)", who);
  return MFN_OK;
}

long long census_parts(int H, int W) {
  return (long long)((H + mfn::unsup::TH - 1) / mfn::unsup::TH) * ((W + mfn::unsup::TW - 1) / mfn::unsup::TW);
}
long long smoothness_parts(int H, int W) { return ((long long)H * W + mfn::unsup::SNT - 1) / mfn::unsup::SNT; }
}  // namespace

extern "C" int mfn_census_loss_forward(const float* img1, const float* img2w, const unsigned char* occ, float* coef,
                                       float* vsum, float* loss, void* ws, long long ws_bytes, int N, int H, int W,
                                       void* stream) {
  using namespace mfn;
  const char* who = "mfn_census_loss_forward";
  MFN_REQUIRE(img1 && img2w && occ && coef && vsum && loss && ws, MFN_ERR_INVALID_ARG, "%s: null pointer", who);
  int rc = check_extents(N, H, W, who);
  if (rc) return rc;
  MFN_REQUIRE(aligned(img1, 4) && aligned(img2w, 4) && aligned(coef, 4) && aligned(vsum, 4) && aligned(loss, 4) &&
                  aligned(ws, 4),
              MFN_ERR_INVALID_ARG, "%s: float pointers must be 4-byte aligned", who);
  const long long parts = census_parts(H, W);
  MFN_REQUIRE(ws_bytes >= 8 * (long long)N * parts, MFN_ERR_INVALID_ARG,
              "%s: workspace smaller than 8*N*ceil(H/8)*ceil(W/32) bytes", who);
  cudaStream_t st = as_stream(stream);
  float* partial = static_cast<float*>(ws);
  unsup::census_forward_kernel<<<dim3((W + unsup::TW - 1) / unsup::TW, (H + unsup::TH - 1) / unsup::TH, N), unsup::NT, 0,
                                 st>>>(img1, img2w, occ, coef, partial, H, W);
  rc = check_launch("census_forward_kernel");
  if (rc) return rc;
  unsup::finish_kernel<<<N, unsup::FNT, 0, st>>>(partial, (int)parts, loss, vsum, H, W);
  return check_launch("census_finish_kernel");
}

extern "C" int mfn_census_loss_backward(const float* img1, const float* img2w, const float* coef, const float* vsum,
                                        const float* g_loss, float* g_img2w, int N, int H, int W, void* stream) {
  using namespace mfn;
  const char* who = "mfn_census_loss_backward";
  MFN_REQUIRE(img1 && img2w && coef && vsum && g_loss && g_img2w, MFN_ERR_INVALID_ARG, "%s: null pointer", who);
  int rc = check_extents(N, H, W, who);
  if (rc) return rc;
  MFN_REQUIRE(aligned(img1, 4) && aligned(img2w, 4) && aligned(coef, 4) && aligned(vsum, 4) && aligned(g_loss, 4) &&
                  aligned(g_img2w, 4),
              MFN_ERR_INVALID_ARG, "%s: float pointers must be 4-byte aligned", who);
  unsup::census_backward_kernel<<<dim3((W + unsup::TW - 1) / unsup::TW, (H + unsup::TH - 1) / unsup::TH, N), unsup::NT, 0,
                                  as_stream(stream)>>>(img1, img2w, coef, vsum, g_loss, g_img2w, H, W);
  return check_launch("census_backward_kernel");
}

extern "C" int mfn_smoothness_loss_forward(const float* flow, const float* img, float* loss, void* ws, long long ws_bytes,
                                           int N, int H, int W, void* stream) {
  using namespace mfn;
  const char* who = "mfn_smoothness_loss_forward";
  MFN_REQUIRE(flow && img && loss && ws, MFN_ERR_INVALID_ARG, "%s: null pointer", who);
  int rc = check_extents(N, H, W, who);
  if (rc) return rc;
  MFN_REQUIRE(aligned(flow, 4) && aligned(img, 4) && aligned(loss, 4) && aligned(ws, 4), MFN_ERR_INVALID_ARG,
              "%s: float pointers must be 4-byte aligned", who);
  const long long parts = smoothness_parts(H, W);
  MFN_REQUIRE(ws_bytes >= 8 * (long long)N * parts, MFN_ERR_INVALID_ARG,
              "%s: workspace smaller than 8*N*ceil(H*W/256) bytes", who);
  cudaStream_t st = as_stream(stream);
  float* partial = static_cast<float*>(ws);
  unsup::smoothness_forward_kernel<<<dim3((unsigned)parts, N), unsup::SNT, 0, st>>>(flow, img, partial, H, W);
  rc = check_launch("smoothness_forward_kernel");
  if (rc) return rc;
  unsup::finish_kernel<<<N, unsup::FNT, 0, st>>>(partial, (int)parts, loss, nullptr, H, W);
  return check_launch("smoothness_finish_kernel");
}

extern "C" int mfn_smoothness_loss_backward(const float* flow, const float* img, const float* g_loss, float* g_flow, int N,
                                            int H, int W, void* stream) {
  using namespace mfn;
  const char* who = "mfn_smoothness_loss_backward";
  MFN_REQUIRE(flow && img && g_loss && g_flow, MFN_ERR_INVALID_ARG, "%s: null pointer", who);
  int rc = check_extents(N, H, W, who);
  if (rc) return rc;
  MFN_REQUIRE(aligned(flow, 4) && aligned(img, 4) && aligned(g_loss, 4) && aligned(g_flow, 4), MFN_ERR_INVALID_ARG,
              "%s: float pointers must be 4-byte aligned", who);
  unsup::smoothness_backward_kernel<<<dim3((unsigned)smoothness_parts(H, W), N), unsup::SNT, 0, as_stream(stream)>>>(
      flow, img, g_loss, g_flow, H, W);
  return check_launch("smoothness_backward_kernel");
}
#endif  // !MFN_HOST_EMULATION
