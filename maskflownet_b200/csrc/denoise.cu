// denoise.cu -- temporal video denoising along the flow, and a noise estimate.
//
//   mfn_denoise_frames   frames ring (S,H,W,3) uint8, flow_fw / flow_bw rings (S,H,W,2)  ->  out (N,H,W,3) uint8
//     denoise_kernel, grid (tiles, 1, N), 16 x 16 threads: one CTA per 16 x 16 output tile of one frame.  The CTA walks
//     the trajectories of the tile and an r-pixel halo around it (the patch radius), one chain step k at a time: each
//     halo position's chain state and its aligned colour a_k sit in shared memory, and after a barrier every tile pixel
//     forms its patch distance from its neighbours' aligned colours and adds the weighted colour to its sums, which stay
//     in registers.  No aligned-frame buffer, no atomics: deterministic.
//   mfn_noise_sigma      frames (F,H,W,3) uint8  ->  sigma (F) float64
//     noise_sigma_kernel, grid F, 1024 threads: int64 sums of |Laplacian-difference filter| per thread, a fixed tree.
// The rules are in include/maskflow_b200.h ("Video denoising").
//
// The file also builds for the host (MFN_HOST_EMULATION: tests/host_emu/denoise_emu.cpp): the kernels are composed of
// per-thread device functions that the emulation calls in the same order, with the barriers in between.
#ifdef MFN_HOST_EMULATION
#include "cuda_shim.h"
#else
#include <math.h>

#include "common.cuh"
#endif
#include "flowcheck.cuh"   // fb_sample, fb_consistent, fb_lerp

namespace mfn {

constexpr int kDnTile = 16;
constexpr int kDnThreads = kDnTile * kDnTile;
constexpr int kDnMaxPatch = 8;          // (16 + 2 r)^2 positions x 32 B of shared memory: 32 KiB at r = 8
constexpr int kNoiseThreads = 1024;

struct DnArgs {
  const unsigned char* frames;           // (S,H,W,3)
  const float2* fw;                      // (S,H,W): slot t mod S holds pair (t, t+1), t -> t+1
  const float2* bw;                      //          ... t+1 -> t
  unsigned char* out;                    // (N,H,W,3)
  int S, H, W, t0, t_lo, t_hi, R, r;
  float alpha, beta, two_s2, h2;         // 2 sigma^2 and (h_factor sigma)^2, both in float32
};

__host__ __device__ inline int dn_halo(int r) { return kDnTile + 2 * r; }
__host__ __device__ inline size_t dn_slot(int t, int S) { return (size_t)(t % S); }

// shared memory of the CTA, P = (16 + 2r)^2 positions, planes of P floats: qx, qy (the chain's position, NaN once it has
// stopped or outside the frame), a_k (3 planes, NaN where undefined), I_t (3 planes)
struct DnShared {
  float *qx, *qy, *col, *ref;
  int P, Hh;
};
__host__ __device__ inline DnShared dn_shared(float* sm, int r) {
  DnShared s;
  s.Hh = dn_halo(r);
  s.P = s.Hh * s.Hh;
  s.qx = sm;
  s.qy = sm + s.P;
  s.col = sm + 2 * s.P;
  s.ref = sm + 5 * s.P;
  return s;
}

// halo position i of the tile whose top-left pixel is (bx0, by0): the chain starts at p, and I_t(p) is loaded
__device__ __forceinline__ void dn_start(const DnArgs& a, int t, int bx0, int by0, int i, DnShared s) {
  const float nan = __int_as_float(0x7fc00000);
  const int hy = i / s.Hh, hx = i - hy * s.Hh;
  const int x = bx0 - a.r + hx, y = by0 - a.r + hy;
  if (x >= 0 && x < a.W && y >= 0 && y < a.H) {
    s.qx[i] = (float)x;
    s.qy[i] = (float)y;
    const unsigned char* p = a.frames + (dn_slot(t, a.S) * a.H * a.W + (size_t)y * a.W + x) * 3;
    for (int c = 0; c < 3; ++c) s.ref[c * s.P + i] = (float)__ldg(p + c);
  } else {
    s.qx[i] = nan;
    s.qy[i] = nan;
    for (int c = 0; c < 3; ++c) s.ref[c * s.P + i] = 0.f;
  }
}

// step k of the chain of halo position i towards frame u = t + k (fwd) or t - k: the step plane, the check plane, the
// colour of frame u at the new position (bilinear, fb_sample's corner rule), or NaN everywhere once the chain stops.
__device__ __forceinline__ void dn_step(const DnArgs& a, int t, int k, bool fwd, int i, DnShared s) {
  const float nan = __int_as_float(0x7fc00000);
  const float qx = s.qx[i], qy = s.qy[i];
  bool live = qx == qx;
  float nx = nan, ny = nan;
  const size_t HW = (size_t)a.H * a.W;
  if (live) {
    const size_t pair = dn_slot(fwd ? t + k - 1 : t - k, a.S) * HW;
    const float2* step = (fwd ? a.fw : a.bw) + pair;
    const float2* check = (fwd ? a.bw : a.fw) + pair;
    const float2 w = fb_sample(step, a.H, a.W, qx, qy);
    nx = qx + w.x;
    ny = qy + w.y;
    live = nx >= 0.f && nx <= (float)(a.W - 1) && ny >= 0.f && ny <= (float)(a.H - 1) &&
           fb_consistent(w, fb_sample(check, a.H, a.W, nx, ny), a.alpha, a.beta);
  }
  if (!live) {
    s.qx[i] = nan;
    s.qy[i] = nan;
    for (int c = 0; c < 3; ++c) s.col[c * s.P + i] = nan;
    return;
  }
  s.qx[i] = nx;
  s.qy[i] = ny;
  const int x0 = (int)floorf(nx), y0 = (int)floorf(ny);
  const int x1 = min(x0 + 1, a.W - 1), y1 = min(y0 + 1, a.H - 1);
  const float wx = nx - (float)x0, wy = ny - (float)y0;
  const unsigned char* img = a.frames + dn_slot(fwd ? t + k : t - k, a.S) * HW * 3;
  const unsigned char* pa = img + 3 * ((size_t)y0 * a.W + x0);
  const unsigned char* pb = img + 3 * ((size_t)y0 * a.W + x1);
  const unsigned char* pc = img + 3 * ((size_t)y1 * a.W + x0);
  const unsigned char* pd = img + 3 * ((size_t)y1 * a.W + x1);
  for (int c = 0; c < 3; ++c)
    s.col[c * s.P + i] = fb_lerp(fb_lerp((float)__ldg(pa + c), (float)__ldg(pb + c), wx),
                                 fb_lerp((float)__ldg(pc + c), (float)__ldg(pd + c), wx), wy);
}

// tile pixel (tx, ty), inside the frame: the patch weight of the current neighbour and its share of the sums
// acc = (sum w, sum w a_0, sum w a_1, sum w a_2)
__device__ __forceinline__ void dn_accumulate(const DnArgs& a, int tx, int ty, DnShared s, float acc[4]) {
  const int ci = (ty + a.r) * s.Hh + tx + a.r;
  const float c0 = s.col[ci];
  if (!(c0 == c0)) return;   // a_k(p) undefined: w = 0
  float D = 0.f;
  int n = 0;
  for (int oy = -a.r; oy <= a.r; ++oy)
    for (int ox = -a.r; ox <= a.r; ++ox) {
      const int j = ci + oy * s.Hh + ox;
      if (!(s.col[j] == s.col[j])) continue;   // outside the frame or not defined
      ++n;
      for (int c = 0; c < 3; ++c) {
        const float d = s.col[c * s.P + j] - s.ref[c * s.P + j];
        D += d * d;
      }
    }
  const float d2 = D / (float)(3 * n);
  const float w = expf(-fmaxf(d2 - a.two_s2, 0.f) / a.h2);
  acc[0] += w;
  for (int c = 0; c < 3; ++c) acc[1 + c] += w * s.col[c * s.P + ci];
}

// out(p) = rint((I_t(p) + sum w a) / (1 + sum w)) per channel, clamped to [0,255]
__device__ __forceinline__ void dn_store(const DnArgs& a, int t, int n, int x, int y, const float acc[4]) {
  const size_t HW = (size_t)a.H * a.W, pix = (size_t)y * a.W + x;
  const unsigned char* src = a.frames + (dn_slot(t, a.S) * HW + pix) * 3;
  unsigned char* o = a.out + ((size_t)n * HW + pix) * 3;
  const float den = 1.f + acc[0];
  for (int c = 0; c < 3; ++c) {
    const float v = rintf(((float)__ldg(src + c) + acc[1 + c]) / den);
    o[c] = (unsigned char)fminf(fmaxf(v, 0.f), 255.f);
  }
}

// the chain length of one direction for frame t
__host__ __device__ inline int dn_steps(const DnArgs& a, int t, bool fwd) {
  const int room = fwd ? a.t_hi - t : t - a.t_lo;
  return room < a.R ? room : a.R;
}

#ifndef MFN_HOST_EMULATION
// grid (tiles_x * tiles_y, 1, N), block (16, 16), 8 P floats of dynamic shared memory
__global__ void __launch_bounds__(kDnThreads) denoise_kernel(DnArgs a, int tiles_x) {
  extern __shared__ float sm[];
  const DnShared s = dn_shared(sm, a.r);
  const int tid = threadIdx.y * kDnTile + threadIdx.x;
  const int n = blockIdx.z, t = a.t0 + n;
  const int by = blockIdx.x / tiles_x, bx = blockIdx.x - by * tiles_x;
  const int bx0 = bx * kDnTile, by0 = by * kDnTile;
  const int x = bx0 + threadIdx.x, y = by0 + threadIdx.y;
  const bool inside = x < a.W && y < a.H;
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
  for (int dir = 0; dir < 2; ++dir) {
    const bool fwd = dir == 0;
    const int K = dn_steps(a, t, fwd);   // the same for the whole CTA
    if (K <= 0) continue;
    __syncthreads();   // the previous direction's last accumulation has read the shared planes
    for (int i = tid; i < s.P; i += kDnThreads) dn_start(a, t, bx0, by0, i, s);
    for (int k = 1; k <= K; ++k) {
      for (int i = tid; i < s.P; i += kDnThreads) dn_step(a, t, k, fwd, i, s);
      __syncthreads();
      if (inside) dn_accumulate(a, threadIdx.x, threadIdx.y, s, acc);
      __syncthreads();
    }
  }
  if (inside) dn_store(a, t, n, x, y, acc);
}
#endif  // !MFN_HOST_EMULATION

// ---- noise estimate -------------------------------------------------------------------------------------------------
// thread t of T: the sum over its interior pixels i = t, t + T, ... (row-major over the (H-2) x (W-2) interior) and the
// three channels of |I * [[1,-2,1],[-2,4,-2],[1,-2,1]]|, exact in int64
__device__ __forceinline__ long long noise_thread_sum(const unsigned char* __restrict__ f, int H, int W, int t, int T) {
  const unsigned IW = (unsigned)(W - 2), n = (unsigned)(H - 2) * IW;   // < 2^31
  long long sum = 0;
  for (unsigned i = (unsigned)t; i < n; i += (unsigned)T) {
    const int y = (int)(i / IW) + 1, x = (int)(i - (unsigned)(y - 1) * IW) + 1;
    const unsigned char* m = f + 3 * ((size_t)y * W + x);
    const unsigned char* u = m - 3 * (size_t)W;
    const unsigned char* d = m + 3 * (size_t)W;
    for (int c = 0; c < 3; ++c) {
      const int v = (int)__ldg(u - 3 + c) - 2 * (int)__ldg(u + c) + (int)__ldg(u + 3 + c) - 2 * (int)__ldg(m - 3 + c) +
                    4 * (int)__ldg(m + c) - 2 * (int)__ldg(m + 3 + c) + (int)__ldg(d - 3 + c) - 2 * (int)__ldg(d + c) +
                    (int)__ldg(d + 3 + c);
      sum += v < 0 ? -v : v;
    }
  }
  return sum;
}

// one level of the fixed reduction tree over kNoiseThreads slots
__device__ __forceinline__ void noise_tree_step(long long* sh, int t, int stride) {
  if (t < stride) sh[t] += sh[t + stride];
}

// sigma = sqrt(pi/2) S / (18 (W-2) (H-2)) in float64, floored at kNoiseFloor
constexpr double kNoiseFloor = 0.5;
__host__ __device__ inline double noise_sigma_of(long long S, int H, int W) {
  const double s = 1.2533141373155003 * (double)S / (18.0 * (double)(W - 2) * (double)(H - 2));
  return s < kNoiseFloor ? kNoiseFloor : s;
}

#ifndef MFN_HOST_EMULATION
__global__ void __launch_bounds__(kNoiseThreads)
    noise_sigma_kernel(const unsigned char* __restrict__ frames, double* __restrict__ sigma, int H, int W) {
  __shared__ long long sh[kNoiseThreads];
  const int t = threadIdx.x;
  const size_t f = blockIdx.x;
  sh[t] = noise_thread_sum(frames + f * 3 * (size_t)H * W, H, W, t, kNoiseThreads);
  __syncthreads();
  for (int stride = kNoiseThreads / 2; stride > 0; stride >>= 1) {
    noise_tree_step(sh, t, stride);
    __syncthreads();
  }
  if (t == 0) sigma[f] = noise_sigma_of(sh[0], H, W);
}
#endif  // !MFN_HOST_EMULATION

}  // namespace mfn

#ifndef MFN_HOST_EMULATION
namespace {
bool dn_positive_finite(float v) { return v > 0.f && v <= 3.402823466e38f; }
bool dn_finite_nonneg(float v) { return v >= 0.f && v <= 3.402823466e38f; }
}  // namespace

extern "C" int mfn_denoise_frames(const unsigned char* frames, const float* flow_fw, const float* flow_bw,
                                  unsigned char* out, int S, int H, int W, int t0, int N, int t_lo, int t_hi,
                                  int radius, int patch, float sigma, float h_factor, float alpha, float beta,
                                  void* stream) {
  using namespace mfn;
  MFN_REQUIRE(frames && flow_fw && flow_bw && out, MFN_ERR_INVALID_ARG, "mfn_denoise_frames: null pointer");
  MFN_REQUIRE(S > 0 && H > 0 && W > 0 && N > 0, MFN_ERR_INVALID_ARG, "mfn_denoise_frames: non-positive extent");
  MFN_REQUIRE(radius >= 0 && patch >= 0, MFN_ERR_INVALID_ARG,
              "mfn_denoise_frames: radius and patch must be >= 0, got %d, %d", radius, patch);
  MFN_REQUIRE(dn_positive_finite(sigma) && dn_positive_finite(h_factor), MFN_ERR_INVALID_ARG,
              "mfn_denoise_frames: sigma and h_factor must be positive and finite, got %g, %g", (double)sigma,
              (double)h_factor);
  MFN_REQUIRE(dn_finite_nonneg(alpha) && dn_finite_nonneg(beta), MFN_ERR_INVALID_ARG,
              "mfn_denoise_frames: alpha and beta must be finite and non-negative");
  const long long first = t0, last = (long long)t0 + N - 1;
  MFN_REQUIRE(t_lo >= 0 && t_lo <= first && last <= t_hi, MFN_ERR_INVALID_ARG,
              "mfn_denoise_frames: frames %lld..%lld outside the video's frames %d..%d", first, last, t_lo, t_hi);
  const long long lo = first - radius > t_lo ? first - radius : t_lo;
  const long long hi = last + radius < t_hi ? last + radius : t_hi;
  MFN_REQUIRE(hi - lo + 1 <= S, MFN_ERR_INVALID_ARG,
              "mfn_denoise_frames: the windows span frames %lld..%lld, more than the ring's %d slots", lo, hi, S);
  MFN_REQUIRE(aligned(flow_fw, 8) && aligned(flow_bw, 8), MFN_ERR_INVALID_ARG,
              "mfn_denoise_frames: flow_fw and flow_bw must be 8-byte aligned");
  MFN_REQUIRE((long long)H * W < (1LL << 31) && N <= 65535, MFN_ERR_ALIGNMENT,
              "mfn_denoise_frames: extents overflow kernel indexing");
  MFN_REQUIRE(patch <= kDnMaxPatch, MFN_ERR_UNSUPPORTED, "mfn_denoise_frames: patch radius %d above %d", patch,
              kDnMaxPatch);
  DnArgs a;
  a.frames = frames;
  a.fw = reinterpret_cast<const float2*>(flow_fw);
  a.bw = reinterpret_cast<const float2*>(flow_bw);
  a.out = out;
  a.S = S, a.H = H, a.W = W, a.t0 = t0, a.t_lo = t_lo, a.t_hi = t_hi, a.R = radius, a.r = patch;
  a.alpha = alpha, a.beta = beta;
  a.two_s2 = 2.f * (sigma * sigma);
  const float hs = h_factor * sigma;
  a.h2 = hs * hs;
  const int tiles_x = (W + kDnTile - 1) / kDnTile, tiles_y = (H + kDnTile - 1) / kDnTile;
  const size_t smem = sizeof(float) * 8 * (size_t)dn_halo(patch) * dn_halo(patch);
  denoise_kernel<<<dim3((unsigned)tiles_x * tiles_y, 1, N), dim3(kDnTile, kDnTile), smem, as_stream(stream)>>>(a,
                                                                                                                tiles_x);
  return check_launch("denoise_kernel");
}

extern "C" int mfn_noise_sigma(const unsigned char* frames, double* sigma, int F, int H, int W, void* stream) {
  using namespace mfn;
  MFN_REQUIRE(frames && sigma, MFN_ERR_INVALID_ARG, "mfn_noise_sigma: null pointer");
  MFN_REQUIRE(F > 0, MFN_ERR_INVALID_ARG, "mfn_noise_sigma: non-positive extent");
  MFN_REQUIRE(H >= 3 && W >= 3, MFN_ERR_INVALID_ARG, "mfn_noise_sigma: frames of %d x %d have no interior pixel", H, W);
  MFN_REQUIRE(aligned(sigma, 8), MFN_ERR_INVALID_ARG, "mfn_noise_sigma: sigma must be 8-byte aligned");
  MFN_REQUIRE((long long)H * W < (1LL << 31) && F <= 65535, MFN_ERR_ALIGNMENT,
              "mfn_noise_sigma: extents overflow kernel indexing");
  noise_sigma_kernel<<<F, kNoiseThreads, 0, as_stream(stream)>>>(frames, sigma, H, W);
  return check_launch("noise_sigma_kernel");
}
#endif  // !MFN_HOST_EMULATION
