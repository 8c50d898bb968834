// augment.cu -- the reference's GPU-side training augmentation (SURVEY.md section 8f, row N4), fused:
//
//   mfn_geometry_augment_forward  replaces GeometryAugmentation.hybrid_forward (augmentation.py:278-339): the reference builds
//       two affine grids (GridGenerator), their common forced translation (two full-grid max / min reductions), a 6-channel
//       concat(img1, mask, flow * mask), two BilinearSampler passes, the mask division, two batch_dot's over the flow and an
//       identity-grid term -- ~25 operator launches and ~10 full-size temporaries.  Here: ONE launch, one thread per target
//       pixel, no temporaries; `/ 255` of train_batch (network/pipeline.py:100) folded into the taps.
//   mfn_color_augment_forward     replaces ColorAugmentation.hybrid_forward (augmentation.py:182-227) for both images: hue /
//       saturation matrix, additive noise, per-image per-channel mean, contrast x channel gain, optional spin matrix,
//       brightness, clip, gamma -- two launches (partial sums of the pre-mean image; apply), the noise either read from a
//       caller tensor or generated in the kernel (Philox4x32-10, counter = pixel, so that both passes see the same value).
//
// The random DRAWS are host logic (maskflownet_b200/augment.py derives the per-sample parameter blocks exactly as the
// reference derives its matrices); the kernels are deterministic functions of (inputs, parameter block).
// Grid arithmetic is written with explicit round-to-nearest intrinsics in the oracle's order (oracle/augment_ref.py), so
// that the forced translation -- a max / min over the grid, evaluated here at the four corners, where a monotone affine
// map in floating point takes its extremes -- is the same number the reference's full reduction produces.
//
// MFN_HOST_EMULATION: the development container has no GPU, so tests/host_emu/ compiles THIS file with g++ behind a small
// shim (threads run one after the other) and tests/test_host_logic.py checks the kernels' arithmetic against the oracle on
// the CPU -- test infrastructure for the kernel source, never a product path (the shim has no launcher, no C ABI).
#ifdef MFN_HOST_EMULATION
#include "cuda_shim.h"
#include "device_caps.h"
#else
#include "common.cuh"
#endif

namespace mfn {
namespace aug {

constexpr int GEO_P = 22;   // floats per sample: affine_params[6], affine_2[6], rel_translation[2], inverse_2[4], factor[4]
constexpr int COL_P = 26;   // sh_matrix[9], contrast*channel[3], channel[3], brightness, pow exponent, spin_matrix[9]
constexpr int SLICES = 64;  // partial sums per (image, sample)

__device__ __forceinline__ float affine_at(float a, float b, float c, float xs, float ys) {
  return __fadd_rn(__fadd_rn(__fmul_rn(a, xs), __fmul_rn(b, ys)), c);
}

// max(grid.max - 1, 0) + min(grid.min + 1, 0) of the affine grid (augmentation.py:311), from its four corners
__device__ __forceinline__ float forced_translation(float a, float b, float c, float x1, float y1) {
  const float v00 = affine_at(a, b, c, -1.f, -1.f), v01 = affine_at(a, b, c, x1, -1.f);
  const float v10 = affine_at(a, b, c, -1.f, y1), v11 = affine_at(a, b, c, x1, y1);
  const float mx = fmaxf(fmaxf(v00, v01), fmaxf(v10, v11)), mn = fminf(fminf(v00, v01), fminf(v10, v11));
  return __fadd_rn(fmaxf(__fadd_rn(mx, -1.f), 0.f), fminf(__fadd_rn(mn, 1.f), 0.f));
}

// MXNet BilinearSampler taps (bilinear_sampler-inl.h restated in oracle/mfn_oracle.c): corners outside the image weigh 0
struct Taps {
  int o00, o01, o10, o11;
  float w00, w01, w10, w11;
};
__device__ __forceinline__ Taps sampler_taps(float gx, float gy, int H, int W) {
  const float xr = __fdiv_rn(__fmul_rn(__fadd_rn(gx, 1.f), (float)(W - 1)), 2.f);
  const float yr = __fdiv_rn(__fmul_rn(__fadd_rn(gy, 1.f), (float)(H - 1)), 2.f);
  const float fx = floorf(xr), fy = floorf(yr);
  // positions far outside contribute nothing; clamping first keeps the float -> int conversion defined for any parameters
  const bool far = !(xr > -2.f && xr < (float)(W + 1) && yr > -2.f && yr < (float)(H + 1));
  const int x0 = far ? -4 : (int)fx, y0 = far ? -4 : (int)fy;
  const float wx0 = __fsub_rn(1.f, __fsub_rn(xr, fx)), wy0 = __fsub_rn(1.f, __fsub_rn(yr, fy));
  const float wx1 = __fsub_rn(1.f, wx0), wy1 = __fsub_rn(1.f, wy0);
  const bool cx0 = x0 >= 0 && x0 <= W - 1, cx1 = x0 + 1 >= 0 && x0 + 1 <= W - 1;
  const bool cy0 = y0 >= 0 && y0 <= H - 1, cy1 = y0 + 1 >= 0 && y0 + 1 <= H - 1;
  const int xa = min(max(x0, 0), W - 1), xb = min(max(x0 + 1, 0), W - 1);
  const int ya = min(max(y0, 0), H - 1), yb = min(max(y0 + 1, 0), H - 1);
  Taps t;
  t.o00 = ya * W + xa;
  t.o01 = ya * W + xb;
  t.o10 = yb * W + xa;
  t.o11 = yb * W + xb;
  t.w00 = (cx0 && cy0 && !far) ? __fmul_rn(wy0, wx0) : 0.f;
  t.w01 = (cx1 && cy0 && !far) ? __fmul_rn(wy0, wx1) : 0.f;
  t.w10 = (cx0 && cy1 && !far) ? __fmul_rn(wy1, wx0) : 0.f;
  t.w11 = (cx1 && cy1 && !far) ? __fmul_rn(wy1, wx1) : 0.f;
  return t;
}

// uint8 sources are read as value / 255 (network/pipeline.py:100).  The 28 taps of a pixel would cost 28 IEEE divisions
// (~10 instructions each; the first version of the kernel spent most of its issue slots there): the 256 possible quotients are tabulated once per block instead --
// the same correctly rounded values, one shared-memory load per tap.
template <typename T>
__device__ __forceinline__ float ld(const T* p, int o, const float* lut) {
  return lut[__ldg(p + o)];
}
template <>
__device__ __forceinline__ float ld<float>(const float* p, int o, const float*) {
  return __ldg(p + o);
}

// one thread per target pixel.  T = element type of the images and the mask: unsigned char (values / 255) or float.
template <typename T>
__global__ void __launch_bounds__(256)
    geometry_augment_kernel(const T* __restrict__ img1, const T* __restrict__ img2, const float* __restrict__ flow,
                            const T* __restrict__ mask, int mask_broadcast, const float* __restrict__ params,
                            float* __restrict__ o1, float* __restrict__ o2, float* __restrict__ of, float* __restrict__ om, int N,
                            int H, int W, int TH, int TW, float sx, float sy, float divisor) {
  const int tplane = TH * TW;
  const size_t plane = (size_t)H * W;
  const long long total = (long long)N * tplane;
  const float x1 = __fadd_rn(-1.f, __fmul_rn((float)(TW - 1), sx)), y1 = __fadd_rn(-1.f, __fmul_rn((float)(TH - 1), sy));
  const float half_w = (float)(0.5 * (double)(W - 1)), half_h = (float)(0.5 * (double)(H - 1));
  __shared__ float div[256];
  if (sizeof(T) == 1) {
    for (int v = threadIdx.x; v < 256; v += blockDim.x) div[v] = __fdiv_rn((float)v, divisor);
    __syncthreads();
  }
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    const int n = (int)(idx / tplane), rem = (int)(idx - (long long)n * tplane);
    const int ty = rem / TW, tx = rem - ty * TW;
    const float* P = params + (size_t)n * GEO_P;
    const float xs = __fadd_rn(-1.f, __fmul_rn((float)tx, sx)), ys = __fadd_rn(-1.f, __fmul_rn((float)ty, sy));
    const float a0 = __ldg(P + 0), a1 = __ldg(P + 1), a2 = __ldg(P + 2), a3 = __ldg(P + 3), a4 = __ldg(P + 4), a5 = __ldg(P + 5);
    const float ftx = forced_translation(a0, a1, a2, x1, y1), fty = forced_translation(a3, a4, a5, x1, y1);
    const float rtx = __ldg(P + 12), rty = __ldg(P + 13);
    // ---- first image, mask, flow: grid clipped into the source image (augmentation.py:310-318) ----
    const float gx = fminf(fmaxf(__fsub_rn(affine_at(a0, a1, a2, xs, ys), ftx), -1.f), 1.f);
    const float gy = fminf(fmaxf(__fsub_rn(affine_at(a3, a4, a5, xs, ys), fty), -1.f), 1.f);
    const Taps t = sampler_taps(gx, gy, H, W);
    const T* p1 = img1 + (size_t)n * 3 * plane;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const T* q = p1 + (size_t)c * plane;
      float v = 0.f;
      v += ld(q, t.o00, div) * t.w00;
      v += ld(q, t.o01, div) * t.w01;
      v += ld(q, t.o10, div) * t.w10;
      v += ld(q, t.o11, div) * t.w11;
      o1[((size_t)n * 3 + c) * tplane + rem] = v;
    }
    float m00, m01, m10, m11;
    if (mask_broadcast) {
      m00 = m01 = m10 = m11 = ld(mask, n, div);
    } else {
      const T* pm = mask + (size_t)n * plane;
      m00 = ld(pm, t.o00, div);
      m01 = ld(pm, t.o01, div);
      m10 = ld(pm, t.o10, div);
      m11 = ld(pm, t.o11, div);
    }
    float mv = 0.f;
    mv += m00 * t.w00;
    mv += m01 * t.w01;
    mv += m10 * t.w10;
    mv += m11 * t.w11;
    om[(size_t)n * tplane + rem] = mv;
    // flow - rel_translation * rel_scale, times the mask, sampled; divided by the sampled mask (:303-307, :318)
    const float shx = __fmul_rn(rtx, half_w), shy = __fmul_rn(rty, half_h);
    const float* pf = flow + (size_t)n * 2 * plane;
    float f[2];
#pragma unroll
    for (int c = 0; c < 2; ++c) {
      const float* q = pf + (size_t)c * plane;
      const float sh = c == 0 ? shx : shy;
      float v = 0.f;
      v += __fmul_rn(__fsub_rn(__ldg(q + t.o00), sh), m00) * t.w00;
      v += __fmul_rn(__fsub_rn(__ldg(q + t.o01), sh), m01) * t.w01;
      v += __fmul_rn(__fsub_rn(__ldg(q + t.o10), sh), m10) * t.w10;
      v += __fmul_rn(__fsub_rn(__ldg(q + t.o11), sh), m11) * t.w11;
      f[c] = __fdiv_rn(v, fmaxf(mv, 1e-8f));
    }
    // flow' = inverse_2 . flow + factor . (x, y) of the identity grid (:326-339)
    const float r0 = __ldg(P + 14) * f[0] + __ldg(P + 15) * f[1] + (__ldg(P + 18) * xs + __ldg(P + 19) * ys);
    const float r1 = __ldg(P + 16) * f[0] + __ldg(P + 17) * f[1] + (__ldg(P + 20) * xs + __ldg(P + 21) * ys);
    of[((size_t)n * 2 + 0) * tplane + rem] = r0;
    of[((size_t)n * 2 + 1) * tplane + rem] = r1;
    // ---- second image: relative transform, same forced translation, zero padding outside (:321-324) ----
    const float g2x = __fadd_rn(__fsub_rn(affine_at(__ldg(P + 6), __ldg(P + 7), __ldg(P + 8), xs, ys), ftx), rtx);
    const float g2y = __fadd_rn(__fsub_rn(affine_at(__ldg(P + 9), __ldg(P + 10), __ldg(P + 11), xs, ys), fty), rty);
    const Taps u = sampler_taps(g2x, g2y, H, W);
    const T* p2 = img2 + (size_t)n * 3 * plane;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const T* q = p2 + (size_t)c * plane;
      float v = 0.f;
      v += ld(q, u.o00, div) * u.w00;
      v += ld(q, u.o01, div) * u.w01;
      v += ld(q, u.o10, div) * u.w10;
      v += ld(q, u.o11, div) * u.w11;
      o2[((size_t)n * 3 + c) * tplane + rem] = v;
    }
  }
}

// ---- counter-based noise: Philox4x32-10 (Salmon et al., SC'11), restated in oracle/augment_ref.py -------------------
__device__ __forceinline__ void philox4x32_10(unsigned c0, unsigned c1, unsigned c2, unsigned c3, unsigned k0, unsigned k1,
                                              unsigned r[4]) {
#pragma unroll
  for (int i = 0; i < 10; ++i) {
    const unsigned h0 = __umulhi(0xD2511F53u, c0), l0 = 0xD2511F53u * c0;
    const unsigned h1 = __umulhi(0xCD9E8D57u, c2), l1 = 0xCD9E8D57u * c2;
    c0 = h1 ^ c1 ^ k0;
    c1 = l1;
    c2 = h0 ^ c3 ^ k1;
    c3 = l0;
    k0 += 0x9E3779B9u;
    k1 += 0xBB67AE85u;
  }
  r[0] = c0;
  r[1] = c1;
  r[2] = c2;
  r[3] = c3;
}
__device__ __forceinline__ float unit_open(unsigned r) { return (float)((r >> 8) + 1u) * 5.9604644775390625e-08f; }   // (0, 1]
__device__ __forceinline__ void normal3(unsigned long long pixel, unsigned image, unsigned long long seed, float z[3]) {
  unsigned r[4];
  philox4x32_10((unsigned)pixel, (unsigned)(pixel >> 32), image, 0u, (unsigned)seed, (unsigned)(seed >> 32), r);
  const float rad0 = sqrtf(-2.f * logf(unit_open(r[0]))), rad1 = sqrtf(-2.f * logf(unit_open(r[2])));
  const float th0 = 6.283185307179586f * unit_open(r[1]), th1 = 6.283185307179586f * unit_open(r[3]);
  z[0] = rad0 * cosf(th0);
  z[1] = rad0 * sinf(th0);
  z[2] = rad1 * cosf(th1);
}

// the image before the mean is taken: sh_matrix . rgb + noise * sigma (augmentation.py:213-215)
__device__ __forceinline__ void pre_mean(const float* __restrict__ img, const float* __restrict__ noise, const float* P,
                                         float sigma, unsigned long long seed, unsigned image, int n, int HW, int pix,
                                         float a[3]) {
  const float* q = img + (size_t)n * 3 * HW + pix;
  const float r = __ldg(q), g = __ldg(q + HW), b = __ldg(q + 2 * (size_t)HW);
#pragma unroll
  for (int i = 0; i < 3; ++i) a[i] = (r * P[3 * i] + g * P[3 * i + 1]) + b * P[3 * i + 2];
  if (noise) {
    const float* nz = noise + (size_t)n * 3 * HW + pix;
#pragma unroll
    for (int i = 0; i < 3; ++i) a[i] += __ldg(nz + (size_t)i * HW) * sigma;
  } else if (sigma != 0.f) {
    float z[3];
    normal3((unsigned long long)n * HW + pix, image, seed, z);
#pragma unroll
    for (int i = 0; i < 3; ++i) a[i] += z[i] * sigma;
  }
}

// grid (SLICES, N, 2 images): partial sums of the three pre-mean channels over a slice of the pixels -> ws[img][n][slice][3]
__global__ void __launch_bounds__(256)
    color_sum_kernel(const float* __restrict__ img1, const float* __restrict__ img2, const float* __restrict__ noise1,
                     const float* __restrict__ noise2, const float* __restrict__ params, float sigma, unsigned long long seed,
                     float* __restrict__ ws, int N, int HW) {
  const int s = blockIdx.x, n = blockIdx.y, image = blockIdx.z;
  const float* img = image ? img2 : img1;
  const float* noise = image ? noise2 : noise1;
  float P[9];
#pragma unroll
  for (int i = 0; i < 9; ++i) P[i] = __ldg(params + (size_t)n * COL_P + i);
  const int beg = (int)((long long)HW * s / SLICES), end = (int)((long long)HW * (s + 1) / SLICES);
  float acc[3] = {0.f, 0.f, 0.f};
  for (int pix = beg + threadIdx.x; pix < end; pix += blockDim.x) {
    float a[3];
    pre_mean(img, noise, P, sigma, seed, (unsigned)image, n, HW, pix, a);
    acc[0] += a[0];
    acc[1] += a[1];
    acc[2] += a[2];
  }
  __shared__ float red[3][8];
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    float v = acc[c];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0) red[c][threadIdx.x >> 5] = v;
  }
  __syncthreads();
  if (threadIdx.x < 3) {
    float v = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) v += red[threadIdx.x][w];
    ws[(((size_t)image * N + n) * SLICES + s) * 3 + threadIdx.x] = v;
  }
}

// grid (blocks per sample, N, 2 images)
__global__ void __launch_bounds__(256)
    color_apply_kernel(const float* __restrict__ img1, const float* __restrict__ img2, const float* __restrict__ noise1,
                       const float* __restrict__ noise2, const float* __restrict__ params, float sigma, unsigned long long seed,
                       const float* __restrict__ ws, float* __restrict__ out1, float* __restrict__ out2, int N, int HW,
                       int has_pow) {
  const int n = blockIdx.y, image = blockIdx.z;
  const float* img = image ? img2 : img1;
  const float* noise = image ? noise2 : noise1;
  float* out = image ? out2 : out1;
  __shared__ float mean_s[3];
  if (threadIdx.x < 3) {
    const float* w = ws + ((size_t)image * N + n) * SLICES * 3 + threadIdx.x;
    float v = 0.f;
    for (int s = 0; s < SLICES; ++s) v += w[3 * s];     // fixed order: deterministic
    mean_s[threadIdx.x] = v / (float)HW;
  }
  __syncthreads();
  float P[COL_P];
#pragma unroll
  for (int i = 0; i < COL_P; ++i) P[i] = __ldg(params + (size_t)n * COL_P + i);
  const float mean[3] = {mean_s[0], mean_s[1], mean_s[2]};
  for (int pix = blockIdx.x * blockDim.x + threadIdx.x; pix < HW; pix += gridDim.x * blockDim.x) {
    float a[3], b[3];
    pre_mean(img, noise, P, sigma, seed, (unsigned)image, n, HW, pix, a);
#pragma unroll
    for (int i = 0; i < 3; ++i) a[i] = (a[i] - mean[i]) * P[9 + i];                            // contrast * channel (:218)
#pragma unroll
    for (int i = 0; i < 3; ++i) b[i] = (a[0] * P[17 + 3 * i] + a[1] * P[18 + 3 * i]) + a[2] * P[19 + 3 * i];   // spin (:220)
#pragma unroll
    for (int i = 0; i < 3; ++i) {
      float v = b[i] + (mean[i] * P[12 + i] + P[15]);                                            // :221
      v = fminf(fmaxf(v, 0.f), 1.f);
      if (has_pow) v = powf(v, P[16]);                                                           // :224
      out[((size_t)n * 3 + i) * HW + pix] = v;
    }
  }
}

static inline unsigned grid_of(long long total) {
  long long b = (total + 255) / 256;
  return (unsigned)(b < 1 ? 1 : (b > (long long)kNumSMs * 32 ? (long long)kNumSMs * 32 : b));
}

}  // namespace aug
}  // namespace mfn

#ifndef MFN_HOST_EMULATION

extern "C" int mfn_geometry_augment_forward(const void* img1, const void* img2, int is_uint8, const float* flow, const void* mask,
                                            int mask_broadcast, const float* params, float* out_img1, float* out_img2,
                                            float* out_flow, float* out_mask, int N, int H, int W, int TH, int TW,
                                            void* stream) {
  using namespace mfn;
  using namespace mfn::aug;
  MFN_REQUIRE(img1 && img2 && flow && mask && params && out_img1 && out_img2 && out_flow && out_mask, MFN_ERR_INVALID_ARG,
              "mfn_geometry_augment_forward: null pointer");
  MFN_REQUIRE(N > 0 && H > 1 && W > 1 && TH > 1 && TW > 1, MFN_ERR_INVALID_ARG,
              "mfn_geometry_augment_forward: extents must be > 1 (the normalised grids divide by extent - 1)");
  MFN_REQUIRE((long long)H * W * 3 < (1LL << 31) && (long long)N * TH * TW < (1LL << 40), MFN_ERR_ALIGNMENT,
              "mfn_geometry_augment_forward: extents overflow kernel indexing");
  const float sx = (float)(2.0 / (double)(TW - 1)), sy = (float)(2.0 / (double)(TH - 1));
  const unsigned grid = grid_of((long long)N * TH * TW);
  cudaStream_t st = as_stream(stream);
  if (is_uint8)
    geometry_augment_kernel<unsigned char><<<grid, 256, 0, st>>>(
        static_cast<const unsigned char*>(img1), static_cast<const unsigned char*>(img2), flow,
        static_cast<const unsigned char*>(mask), mask_broadcast ? 1 : 0, params, out_img1, out_img2, out_flow, out_mask, N, H, W,
        TH, TW, sx, sy, 255.f);
  else
    geometry_augment_kernel<float><<<grid, 256, 0, st>>>(static_cast<const float*>(img1), static_cast<const float*>(img2), flow,
                                                        static_cast<const float*>(mask), mask_broadcast ? 1 : 0, params,
                                                        out_img1, out_img2, out_flow, out_mask, N, H, W, TH, TW, sx, sy, 1.f);
  return check_launch("geometry_augment_kernel");
}

extern "C" long long mfn_color_augment_workspace_bytes(int N) {
  return N > 0 ? (long long)2 * N * mfn::aug::SLICES * 3 * (long long)sizeof(float) : 0;
}

extern "C" int mfn_color_augment_forward(const float* img1, const float* img2, const float* params, const float* noise1,
                                         const float* noise2, float noise_sigma, long long seed, float* out1, float* out2,
                                         void* workspace, long long workspace_bytes, int N, int H, int W, int has_gamma,
                                         void* stream) {
  using namespace mfn;
  using namespace mfn::aug;
  MFN_REQUIRE(img1 && img2 && params && out1 && out2 && workspace, MFN_ERR_INVALID_ARG,
              "mfn_color_augment_forward: null pointer");
  MFN_REQUIRE((noise1 == nullptr) == (noise2 == nullptr), MFN_ERR_INVALID_ARG,
              "mfn_color_augment_forward: pass both noise tensors or neither");
  MFN_REQUIRE(N > 0 && N <= 65535 && H > 0 && W > 0, MFN_ERR_INVALID_ARG, "mfn_color_augment_forward: bad extent");
  MFN_REQUIRE((long long)H * W * 3 < (1LL << 31), MFN_ERR_ALIGNMENT, "mfn_color_augment_forward: image too large");
  MFN_REQUIRE(workspace_bytes >= mfn_color_augment_workspace_bytes(N), MFN_ERR_INVALID_ARG,
              "mfn_color_augment_forward: workspace smaller than mfn_color_augment_workspace_bytes(N)");
  cudaStream_t st = as_stream(stream);
  float* ws = static_cast<float*>(workspace);
  const int HW = H * W;
  color_sum_kernel<<<dim3(SLICES, N, 2), 256, 0, st>>>(img1, img2, noise1, noise2, params, noise_sigma,
                                                       (unsigned long long)seed, ws, N, HW);
  int rc = check_launch("color_sum_kernel");
  if (rc) return rc;
  int bps = (HW + 255) / 256;
  const int cap = (kNumSMs * 16 + 2 * N - 1) / (2 * N);
  if (bps > cap) bps = cap;
  if (bps < 1) bps = 1;
  color_apply_kernel<<<dim3(bps, N, 2), 256, 0, st>>>(img1, img2, noise1, noise2, params, noise_sigma, (unsigned long long)seed,
                                                      ws, out1, out2, N, HW, has_gamma ? 1 : 0);
  return check_launch("color_apply_kernel");
}
#endif  // !MFN_HOST_EMULATION
