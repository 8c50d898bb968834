// corr_bwd.cu -- correlation backward (K2) for sm_90a.
//
// Serves mfn_correlation_backward: the gradient of F.Correlation (network/MaskFlownet.py:193-195, 440-441) that the
// reference obtains implicitly from autograd.record() / loss.backward() (network/pipeline.py:97,112-113).
//
//   g1[n,c,p]  = 1/C * sum_d  go'[q(d)][p]      * f2[c][p+d]
//   g2[n,c,p'] = 1/C * sum_d  go'[q(d)][p'-d]   * f1[c][p'-d]
//              = 1/C * sum_e  T[e][p']          * f1[c][p'+e]      with e = -d,  T[e][p'] = go'[q(-e)][p'+e]
// so both sides are the same stencil "sum_e G[e][p] * X[c][p+e]" and share one kernel; side B gathers its G tile
// through the index map above while loading it.  go' = go * (out > 0 ? 1 : slope) fuses the LeakyReLU backward.
// Gather form on both sides: no atomics, deterministic.
#include "common.cuh"

namespace mfn {
namespace k2 {
// CTA = 4 rows x 32 pixels; thread = one 4-pixel quad x CPT channels (CPT = 1: 56 KB of shared memory, four CTAs per SM --
// measured faster than CPT = 4 with two CTAs per SM: the kernel is bound by the latency of its tile loads, not by the
// shared-memory traffic of the stencil).
constexpr int TH = 4, TW = 32, CPT = 1, CK = 8 * CPT, NT = 256;
}

template <int MD, bool SIDE_B>
__global__ void __launch_bounds__(k2::NT)
    corr_bwd_kernel(const float* __restrict__ go, const float* __restrict__ fwd_out, const float* __restrict__ X,
                    float* __restrict__ gX, int N, int C, int H, int W, long long obs, float slope) {
  using namespace k2;
  constexpr int G = 2 * MD + 1, D = G * G;
  constexpr int HR = TH + 2 * MD, HWD = TW + 8;
  extern __shared__ __align__(16) float smem[];
  float* Gt = smem;                  // [D][TH][TW]
  float* Xs = smem + D * TH * TW;    // [CK][HR][HWD]

  const int tilesX = (W + TW - 1) / TW, tilesY = (H + TH - 1) / TH;
  const int tile = blockIdx.x;
  const int tx = tile % tilesX, ty = (tile / tilesX) % tilesY, n = tile / (tilesX * tilesY);
  const int x0 = tx * TW, y0 = ty * TH;
  const int tid = threadIdx.x;
  const size_t plane = (size_t)H * W;

  const float* gon = go + (size_t)n * obs;
  const float* fon = fwd_out ? fwd_out + (size_t)n * obs : nullptr;
  // G tile: thread (warp w, lane) owns column xx = lane of the tile rows j = w + 8k, j = q * TH + rr  (rr = w & 3 and
  // q = (w >> 2) + 2k).  Loads are issued in batches of 8 before any of them is consumed (a loop that consumes each load
  // at once stalls on that dependency).
  {
    const int w = tid >> 5, xx = tid & 31, rr = w & 3;
    constexpr int KQ = (D + 1) / 2;
#pragma unroll 1
    for (int k0 = 0; k0 < KQ; k0 += 8) {
      float gv[8], fv[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        const int q = (w >> 2) + 2 * (k0 + u);
        gv[u] = 0.f;
        fv[u] = 1.f;
        if (q < D) {
          const int ey = q / G - MD, ex = q % G - MD;
          int ys = y0 + rr, xsrc = x0 + xx, qs = q;
          bool ok = ys < H && xsrc < W;
          if (SIDE_B) {
            qs = (MD - ey) * G + (MD - ex);
            ys += ey;
            xsrc += ex;
            ok = ok && ys >= 0 && ys < H && xsrc >= 0 && xsrc < W;
          }
          if (ok) {
            const size_t i = (size_t)qs * plane + (size_t)ys * W + xsrc;
            gv[u] = __ldg(gon + i);
            if (fon) fv[u] = __ldg(fon + i);
          }
        }
      }
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        const int q = (w >> 2) + 2 * (k0 + u);
        if (q < D) Gt[(q * TH + rr) * TW + xx] = fv[u] > 0.f ? gv[u] : gv[u] * slope;
      }
    }
  }

  const int qx = tid & 7, r = (tid >> 3) & 3, cg = tid >> 5;  // 8 quads x 4 rows x 8 channel groups of CPT
  const float* Xn = X + (size_t)n * C * plane;
  const float inv = 1.f / (float)C;
  for (int c0 = 0; c0 < C; c0 += CK) {
    __syncthreads();
    {   // X tile: warp w owns the rows rho = w + 8k (rho = channel * HR + halo row) of 40 floats: lane -> columns lane and
        // (lanes < 8) 32 + lane; eight rows (16 loads) in flight per thread
      const int w = tid >> 5, lane = tid & 31;
#pragma unroll 1
      constexpr int XB = 4;   // rows per batch: CK * HR / 8 rows per warp (12 or 8 with CPT = 1) in batches of 4
      static_assert((CK * HR / 8) % XB == 0, "row batches");
#pragma unroll
      for (int k0 = 0; k0 < CK * HR / 8; k0 += XB) {
        float va[XB], vb[XB];
#pragma unroll
        for (int u = 0; u < XB; ++u) {
          const int rho = w + 8 * (k0 + u), cc = rho / HR, yy = rho - cc * HR;
          const int c = c0 + cc, y = y0 - MD + yy;
          const bool rok = c < C && y >= 0 && y < H;
          const float* src = Xn + (size_t)c * plane + (size_t)y * W + (x0 - 4);
          const int xa = x0 - 4 + lane, xb = x0 + 28 + lane;
          va[u] = (rok && xa >= 0 && xa < W) ? __ldg(src + lane) : 0.f;
          vb[u] = (rok && lane < 8 && xb < W) ? __ldg(src + 32 + lane) : 0.f;
        }
#pragma unroll
        for (int u = 0; u < XB; ++u) {
          const int rho = w + 8 * (k0 + u);
          Xs[rho * HWD + lane] = va[u];
          if (lane < 8) Xs[rho * HWD + 32 + lane] = vb[u];
        }
      }
    }
    __syncthreads();
    float acc[CPT][4];
#pragma unroll
    for (int k = 0; k < CPT; ++k)
#pragma unroll
      for (int p = 0; p < 4; ++p) acc[k][p] = 0.f;
#pragma unroll
    for (int eyi = 0; eyi < G; ++eyi) {
      float f[CPT][12];
#pragma unroll
      for (int k = 0; k < CPT; ++k) {
        const float* row = Xs + ((cg * CPT + k) * HR + r + eyi) * HWD + 4 * qx;
        const float4 v0 = *reinterpret_cast<const float4*>(row);
        const float4 v1 = *reinterpret_cast<const float4*>(row + 4);
        const float4 v2 = *reinterpret_cast<const float4*>(row + 8);
        f[k][0] = v0.x; f[k][1] = v0.y; f[k][2] = v0.z; f[k][3] = v0.w;
        f[k][4] = v1.x; f[k][5] = v1.y; f[k][6] = v1.z; f[k][7] = v1.w;
        f[k][8] = v2.x; f[k][9] = v2.y; f[k][10] = v2.z; f[k][11] = v2.w;
      }
#pragma unroll
      for (int exi = 0; exi < G; ++exi) {
        const float4 g4 = *reinterpret_cast<const float4*>(Gt + ((eyi * G + exi) * TH + r) * TW + 4 * qx);
#pragma unroll
        for (int k = 0; k < CPT; ++k) {
          acc[k][0] = fmaf(g4.x, f[k][0 + exi + (4 - MD)], acc[k][0]);
          acc[k][1] = fmaf(g4.y, f[k][1 + exi + (4 - MD)], acc[k][1]);
          acc[k][2] = fmaf(g4.z, f[k][2 + exi + (4 - MD)], acc[k][2]);
          acc[k][3] = fmaf(g4.w, f[k][3 + exi + (4 - MD)], acc[k][3]);
        }
      }
    }
    const int y = y0 + r, xb = x0 + 4 * qx;
    if (y < H) {
#pragma unroll
      for (int k = 0; k < CPT; ++k) {
        const int c = c0 + cg * CPT + k;
        if (c >= C) continue;
        float* o = gX + ((size_t)n * C + c) * plane + (size_t)y * W + xb;
        if (xb + 3 < W && (reinterpret_cast<uintptr_t>(o) & 15) == 0) {
          *reinterpret_cast<float4*>(o) = make_float4(acc[k][0] * inv, acc[k][1] * inv, acc[k][2] * inv, acc[k][3] * inv);
        } else {
#pragma unroll
          for (int p = 0; p < 4; ++p)
            if (xb + p < W) o[p] = acc[k][p] * inv;
        }
      }
    }
  }
}

template <int MD>
static int launch_corr_bwd(const float* go, const float* fo, const float* d1, const float* d2, float* g1, float* g2,
                           int N, int C, int H, int W, long long obs, float slope, cudaStream_t st) {
  using namespace k2;
  constexpr int G = 2 * MD + 1, D = G * G;
  const int tilesX = (W + TW - 1) / TW, tilesY = (H + TH - 1) / TH;
  const unsigned tiles = (unsigned)((long long)N * tilesX * tilesY);
  const int smem = (int)sizeof(float) * (D * TH * TW + CK * (TH + 2 * MD) * (TW + 8));
  static SmemOptIn optA, optB;
  cudaError_t ae = ensure_dyn_smem(corr_bwd_kernel<MD, false>, smem, optA);
  if (ae == cudaSuccess) ae = ensure_dyn_smem(corr_bwd_kernel<MD, true>, smem, optB);
  if (ae != cudaSuccess) return fail((int)ae, "cudaFuncSetAttribute(corr_bwd_kernel): %s", cudaGetErrorString(ae));
  if (g1) {
    corr_bwd_kernel<MD, false><<<tiles, NT, smem, st>>>(go, fo, d2, g1, N, C, H, W, obs, slope);
    const int rc = check_launch("corr_bwd_kernel<sideA>");
    if (rc) return rc;
  }
  if (g2) {
    corr_bwd_kernel<MD, true><<<tiles, NT, smem, st>>>(go, fo, d1, g2, N, C, H, W, obs, slope);
    return check_launch("corr_bwd_kernel<sideB>");
  }
  return MFN_OK;
}

}  // namespace mfn

extern "C" int mfn_correlation_backward(const float* grad_out, const float* out, const float* data1,
                                        const float* data2, float* grad1, float* grad2, int N, int C, int H, int W,
                                        int max_displacement, long long out_batch_stride, float leaky_slope,
                                        void* stream) {
  using namespace mfn;
  MFN_REQUIRE(grad_out && data1 && data2 && (grad1 || grad2), MFN_ERR_INVALID_ARG,
              "mfn_correlation_backward: null pointer");
  MFN_REQUIRE(N > 0 && C > 0 && H > 0 && W > 0, MFN_ERR_INVALID_ARG, "mfn_correlation_backward: non-positive extent");
  MFN_REQUIRE(max_displacement == 4 || max_displacement == 2, MFN_ERR_UNSUPPORTED,
              "mfn_correlation_backward: max_displacement must be 4 or 2 (the reference's values), got %d",
              max_displacement);
  const int G = 2 * max_displacement + 1;
  const long long obs = out_batch_stride ? out_batch_stride : (long long)G * G * H * W;
  MFN_REQUIRE(obs >= (long long)G * G * H * W, MFN_ERR_INVALID_ARG, "mfn_correlation_backward: out_batch_stride too small");
  cudaStream_t st = as_stream(stream);
  return max_displacement == 4
             ? launch_corr_bwd<4>(grad_out, out, data1, data2, grad1, grad2, N, C, H, W, obs, leaky_slope, st)
             : launch_corr_bwd<2>(grad_out, out, data1, data2, grad1, grad2, N, C, H, W, obs, leaky_slope, st);
}
