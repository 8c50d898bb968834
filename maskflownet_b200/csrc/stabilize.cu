// stabilize.cu -- video stabilisation: a robust affine camera motion fitted to a dense flow, and a warp of uint8 frames by
// per-frame affine maps.
//
//   mfn_affine_motion        flow (N,H,W,2) (x,y) pixels  ->  affine (N,2,3) float64, ok (N) uint8, residual (N,H,W)
//     per IRLS iteration k (include/maskflow_b200.h states the rule):
//       fit_accumulate_kernel, grid (G, N): each thread sums the 12 weighted moments over a fixed, strided set of pixels in
//       float64, the CTA adds its 256 threads' sums by a fixed shared-memory tree and writes one partial row per CTA;
//       fit_solve_kernel, grid N: one CTA adds the sample's G partial rows in a fixed order, solves the two 3x3 systems
//       and writes affine and ok, which the next iteration's weights read.
//     then, when residual is wanted, fit_residual_kernel, grid (pixels / 256, N).
//     G depends on H x W only, so a sample's fit does not depend on the batch it is in.  No atomics: bit-reproducible.
//   mfn_warp_frames_affine   src (N,H,W,3) uint8, M (N,2,3) float64  ->  out (N,H,W,3) uint8
//     warp_affine_kernel, grid (pixels / 256, N): one thread per output pixel, bilinear in float64.
//
// The file also builds for the host (MFN_HOST_EMULATION: tests/host_emu/stabilize_emu.cpp): the kernels are composed of
// per-thread device functions that the emulation calls in the same order, with the tree steps in between.
#ifdef MFN_HOST_EMULATION
#include "cuda_shim.h"
#else
#include <math.h>

#include "common.cuh"
#endif

namespace mfn {

constexpr int kFitThreads = 256;
constexpr int kFitMoments = 12;   // Sxx Sxy Sx Syy Sy S1 | Sx*qx Sy*qx S1*qx | Sx*qy Sy*qy S1*qy (normalised, weighted)
constexpr int kFitMaxCtas = 256;

// CTAs per sample of the accumulation: about 2048 pixels each, at most kFitMaxCtas
static inline int fit_ctas(int H, int W) {
  const long long HW = (long long)H * W;
  const long long g = (HW + 2047) / 2048;
  return (int)(g < kFitMaxCtas ? g : kFitMaxCtas);
}

// The normalisation of both p and q: centre ((W-1)/2, (H-1)/2), scale max(W,H)/2.
struct FitFrame {
  double cx, cy, s, inv_s;
};
__host__ __device__ inline FitFrame fit_frame(int H, int W) {
  FitFrame f;
  f.cx = 0.5 * (double)(W - 1);
  f.cy = 0.5 * (double)(H - 1);
  f.s = 0.5 * (double)(W > H ? W : H);
  f.inv_s = 1.0 / f.s;
  return f;
}

// Thread t of CTA g (G per sample) of sample n: the moments of pixels p = g * 256 + t + i * G * 256.  A is the previous
// iteration's map in pixels (read when inv_sig2 > 0; 0 selects plain least squares).
__device__ __forceinline__ void fit_thread_sums(const float2* __restrict__ flow, const double* __restrict__ A, int H,
                                                int W, int g, int G, int t, double inv_sig2, double m[kFitMoments]) {
  for (int j = 0; j < kFitMoments; ++j) m[j] = 0.0;
  const FitFrame fr = fit_frame(H, W);
  const unsigned HW = (unsigned)H * (unsigned)W;   // < 2^31, so p + G * 256 cannot wrap
  double a0 = 0, a1 = 0, a2 = 0, a3 = 0, a4 = 0, a5 = 0;
  if (inv_sig2 > 0.0) {
    a0 = A[0], a1 = A[1], a2 = A[2], a3 = A[3], a4 = A[4], a5 = A[5];
  }
  const double xmax = (double)(W - 1), ymax = (double)(H - 1);
  for (unsigned p = (unsigned)g * kFitThreads + t; p < HW; p += (unsigned)G * kFitThreads) {
    const float2 uv = __ldg(flow + p);
    const int y = (int)(p / (unsigned)W), x = (int)(p - (unsigned)y * (unsigned)W);
    const double px = (double)x, py = (double)y;
    const double qx = px + (double)uv.x, qy = py + (double)uv.y;
    if (!(qx >= 0.0 && qx <= xmax && qy >= 0.0 && qy <= ymax)) continue;   // non-finite or outside the frame
    double w = 1.0;
    if (inv_sig2 > 0.0) {
      const double dx = a0 * px + a1 * py + a2 - qx, dy = a3 * px + a4 * py + a5 - qy;
      w = 1.0 / (1.0 + (dx * dx + dy * dy) * inv_sig2);
    }
    const double xh = (px - fr.cx) * fr.inv_s, yh = (py - fr.cy) * fr.inv_s;
    const double ux = (qx - fr.cx) * fr.inv_s, uy = (qy - fr.cy) * fr.inv_s;
    const double wx = w * xh, wy = w * yh;
    m[0] += wx * xh;
    m[1] += wx * yh;
    m[2] += wx;
    m[3] += wy * yh;
    m[4] += wy;
    m[5] += w;
    m[6] += wx * ux;
    m[7] += wy * ux;
    m[8] += w * ux;
    m[9] += wx * uy;
    m[10] += wy * uy;
    m[11] += w * uy;
  }
}

// one level of the fixed reduction tree over 256 slots: slot t < stride adds slot t + stride
__device__ __forceinline__ void fit_tree_step(double (*sh)[kFitMoments], int t, int stride) {
  if (t < stride)
    for (int j = 0; j < kFitMoments; ++j) sh[t][j] += sh[t + stride][j];
}

// Thread t of the solve CTA: the partial rows g = t, t + 256, ... of one sample, added in that order.
__device__ __forceinline__ void fit_partial_sums(const double* __restrict__ part, int G, int t, double m[kFitMoments]) {
  for (int j = 0; j < kFitMoments; ++j) m[j] = 0.0;
  for (int g = t; g < G; g += kFitThreads)
    for (int j = 0; j < kFitMoments; ++j) m[j] += part[(size_t)g * kFitMoments + j];
}

// The two 3x3 solves of the normal equations (adjugate over determinant), the conditioning test and the map back to
// pixels.  A failed solve writes the identity and ok = 0.
__device__ __forceinline__ void fit_solve(const double m[kFitMoments], int H, int W, double* __restrict__ A,
                                          unsigned char* __restrict__ ok) {
  const double a = m[0], b = m[1], c = m[2], d = m[3], e = m[4], f = m[5];
  const double c00 = d * f - e * e, c01 = c * e - b * f, c02 = b * e - c * d;
  const double c11 = a * f - c * c, c12 = b * c - a * e, c22 = a * d - b * b;
  const double det = a * c00 + b * c01 + c * c02;
  const double tr3 = (a + d + f) / 3.0;
  const bool good = f >= 3.0 && det > 1e-9 * tr3 * tr3 * tr3;
  if (!good) {
    A[0] = 1.0, A[1] = 0.0, A[2] = 0.0, A[3] = 0.0, A[4] = 1.0, A[5] = 0.0;
    *ok = 0;
    return;
  }
  const double inv = 1.0 / det;
  double r[2][3];
  for (int k = 0; k < 2; ++k) {
    const double b0 = m[6 + 3 * k], b1 = m[7 + 3 * k], b2 = m[8 + 3 * k];
    r[k][0] = (c00 * b0 + c01 * b1 + c02 * b2) * inv;
    r[k][1] = (c01 * b0 + c11 * b1 + c12 * b2) * inv;
    r[k][2] = (c02 * b0 + c12 * b1 + c22 * b2) * inv;
  }
  const FitFrame fr = fit_frame(H, W);
  A[0] = r[0][0], A[1] = r[0][1], A[2] = fr.cx + fr.s * r[0][2] - (r[0][0] * fr.cx + r[0][1] * fr.cy);
  A[3] = r[1][0], A[4] = r[1][1], A[5] = fr.cy + fr.s * r[1][2] - (r[1][0] * fr.cx + r[1][1] * fr.cy);
  *ok = 1;
}

// grid (G, N), 256 threads: part (N, G, 12) float64
__global__ void __launch_bounds__(kFitThreads, 4)
    fit_accumulate_kernel(const float2* __restrict__ flow, const double* __restrict__ affine, double* __restrict__ part,
                          int H, int W, int G, double inv_sig2) {
  __shared__ double sh[kFitThreads][kFitMoments];
  const int t = threadIdx.x, g = blockIdx.x, n = blockIdx.y;
  double m[kFitMoments];
  fit_thread_sums(flow + (size_t)n * H * W, affine + 6 * n, H, W, g, G, t, inv_sig2, m);
  for (int j = 0; j < kFitMoments; ++j) sh[t][j] = m[j];
  __syncthreads();
  for (int stride = kFitThreads / 2; stride > 0; stride >>= 1) {
    fit_tree_step(sh, t, stride);
    __syncthreads();
  }
  if (t < kFitMoments) part[((size_t)n * G + g) * kFitMoments + t] = sh[0][t];
}

// grid N, 256 threads
__global__ void __launch_bounds__(kFitThreads)
    fit_solve_kernel(const double* __restrict__ part, double* __restrict__ affine, unsigned char* __restrict__ ok, int H,
                     int W, int G) {
  __shared__ double sh[kFitThreads][kFitMoments];
  const int t = threadIdx.x, n = blockIdx.x;
  double m[kFitMoments];
  fit_partial_sums(part + (size_t)n * G * kFitMoments, G, t, m);
  for (int j = 0; j < kFitMoments; ++j) sh[t][j] = m[j];
  __syncthreads();
  for (int stride = kFitThreads / 2; stride > 0; stride >>= 1) {
    fit_tree_step(sh, t, stride);
    __syncthreads();
  }
  if (t == 0) fit_solve(sh[0], H, W, affine + 6 * n, ok + n);
}

// grid (ceil(HW / 256), N): |A p - q| under the final map, NaN where the pixel is not valid
__global__ void __launch_bounds__(256)
    fit_residual_kernel(const float2* __restrict__ flow, const double* __restrict__ affine, float* __restrict__ residual,
                        int H, int W) {
  const int HW = H * W;
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= HW) return;
  const size_t i = (size_t)blockIdx.y * HW + p;
  const double* A = affine + 6 * blockIdx.y;
  const float2 uv = __ldg(flow + i);
  const int y = p / W, x = p - y * W;
  const double px = (double)x, py = (double)y;
  const double qx = px + (double)uv.x, qy = py + (double)uv.y;
  if (!(qx >= 0.0 && qx <= (double)(W - 1) && qy >= 0.0 && qy <= (double)(H - 1))) {
    residual[i] = __int_as_float(0x7fc00000);
    return;
  }
  const double dx = A[0] * px + A[1] * py + A[2] - qx, dy = A[3] * px + A[4] * py + A[5] - qy;
  residual[i] = (float)sqrt(dx * dx + dy * dy);
}

// grid (ceil(HW / 256), N): out(o) = src sampled bilinearly at M o, clamped to the frame
__global__ void __launch_bounds__(256)
    warp_affine_kernel(const unsigned char* __restrict__ src, const double* __restrict__ M, unsigned char* __restrict__ out,
                       int H, int W) {
  const int HW = H * W;
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= HW) return;
  const size_t n = blockIdx.y;
  const double* m = M + 6 * n;
  const int y = p / W, x = p - y * W;
  double sx = m[0] * (double)x + m[1] * (double)y + m[2];
  double sy = m[3] * (double)x + m[4] * (double)y + m[5];
  sx = fmin(fmax(sx, 0.0), (double)(W - 1));   // fmax(NaN, 0) = 0
  sy = fmin(fmax(sy, 0.0), (double)(H - 1));
  const double fx = floor(sx), fy = floor(sy);
  const int x0 = (int)fx, y0 = (int)fy;
  const int x1 = min(x0 + 1, W - 1), y1 = min(y0 + 1, H - 1);
  const double wx = sx - fx, wy = sy - fy;
  const unsigned char* img = src + 3 * n * (size_t)HW;
  const unsigned char* pa = img + 3 * ((size_t)y0 * W + x0);
  const unsigned char* pb = img + 3 * ((size_t)y0 * W + x1);
  const unsigned char* pc = img + 3 * ((size_t)y1 * W + x0);
  const unsigned char* pd = img + 3 * ((size_t)y1 * W + x1);
  unsigned char* o = out + 3 * (n * HW + p);
  for (int c = 0; c < 3; ++c) {
    const double top = (1.0 - wx) * (double)__ldg(pa + c) + wx * (double)__ldg(pb + c);
    const double bot = (1.0 - wx) * (double)__ldg(pc + c) + wx * (double)__ldg(pd + c);
    const double v = rint((1.0 - wy) * top + wy * bot);
    o[c] = (unsigned char)fmin(fmax(v, 0.0), 255.0);
  }
}

}  // namespace mfn

#ifndef MFN_HOST_EMULATION
extern "C" long long mfn_affine_motion_workspace_bytes(int N, int H, int W) {
  return (N > 0 && H > 0 && W > 0) ? 8LL * mfn::kFitMoments * N * mfn::fit_ctas(H, W) : 0;
}

extern "C" int mfn_affine_motion(const float* flow, double* affine, unsigned char* ok, float* residual, void* ws,
                                 long long ws_bytes, int N, int H, int W, int iterations, float sigma, void* stream) {
  using namespace mfn;
  MFN_REQUIRE(flow && affine && ok && ws, MFN_ERR_INVALID_ARG, "mfn_affine_motion: null pointer");
  MFN_REQUIRE(N > 0 && H > 0 && W > 0, MFN_ERR_INVALID_ARG, "mfn_affine_motion: non-positive extent");
  MFN_REQUIRE(iterations >= 1, MFN_ERR_INVALID_ARG, "mfn_affine_motion: iterations must be >= 1, got %d", iterations);
  MFN_REQUIRE(sigma > 0.f && sigma <= 3.402823466e38f, MFN_ERR_INVALID_ARG,
              "mfn_affine_motion: sigma must be positive and finite, got %g", (double)sigma);
  MFN_REQUIRE(aligned(flow, 8) && aligned(affine, 8) && aligned(ws, 8) && aligned(residual, 4), MFN_ERR_INVALID_ARG,
              "mfn_affine_motion: flow, affine and ws must be 8-byte aligned, residual 4-byte aligned");
  MFN_REQUIRE((long long)H * W < (1LL << 31) && N <= 65535, MFN_ERR_ALIGNMENT,
              "mfn_affine_motion: extents overflow kernel indexing");
  const long long need = mfn_affine_motion_workspace_bytes(N, H, W);
  MFN_REQUIRE(ws_bytes >= need, MFN_ERR_INVALID_ARG, "mfn_affine_motion: workspace of %lld bytes, %lld needed", ws_bytes,
              need);
  const int G = fit_ctas(H, W);
  cudaStream_t st = as_stream(stream);
  const float2* f2 = reinterpret_cast<const float2*>(flow);
  double* part = static_cast<double*>(ws);
  for (int k = 0; k < iterations; ++k) {
    // sigma_k = sigma 2^max(0, 4-k): 8 sigma, 4 sigma, 2 sigma, sigma, sigma, ...; iteration 0 is plain least squares
    const double sk = (double)sigma * (double)(1 << (k < 4 ? 4 - k : 0));
    const double inv_sig2 = k == 0 ? 0.0 : 1.0 / (sk * sk);
    fit_accumulate_kernel<<<dim3(G, N), kFitThreads, 0, st>>>(f2, affine, part, H, W, G, inv_sig2);
    if (int rc = check_launch("fit_accumulate_kernel")) return rc;
    fit_solve_kernel<<<N, kFitThreads, 0, st>>>(part, affine, ok, H, W, G);
    if (int rc = check_launch("fit_solve_kernel")) return rc;
  }
  if (residual) {
    const int HW = H * W;
    fit_residual_kernel<<<dim3((HW + 255) / 256, N), 256, 0, st>>>(f2, affine, residual, H, W);
    if (int rc = check_launch("fit_residual_kernel")) return rc;
  }
  return 0;
}

extern "C" int mfn_warp_frames_affine(const unsigned char* src, const double* M, unsigned char* out, int N, int H, int W,
                                      void* stream) {
  using namespace mfn;
  MFN_REQUIRE(src && M && out, MFN_ERR_INVALID_ARG, "mfn_warp_frames_affine: null pointer");
  MFN_REQUIRE(N > 0 && H > 0 && W > 0, MFN_ERR_INVALID_ARG, "mfn_warp_frames_affine: non-positive extent");
  MFN_REQUIRE(aligned(M, 8), MFN_ERR_INVALID_ARG, "mfn_warp_frames_affine: M must be 8-byte aligned");
  MFN_REQUIRE((long long)H * W < (1LL << 31) && N <= 65535, MFN_ERR_ALIGNMENT,
              "mfn_warp_frames_affine: extents overflow kernel indexing");
  const int HW = H * W;
  warp_affine_kernel<<<dim3((HW + 255) / 256, N), 256, 0, as_stream(stream)>>>(src, M, out, H, W);
  return check_launch("warp_affine_kernel");
}
#endif  // !MFN_HOST_EMULATION
