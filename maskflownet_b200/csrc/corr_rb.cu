// corr_rb.cu -- correlation cost-volume forward (K1) for C > 32 (levels 3..6 of the S head and of the cascade) and for the
// shapes the TMA kernel cannot take (W % 4 != 0): "row-block" kernel, sm_90a.
//
// Serves mfn_correlation_forward (include/maskflow_b200.h) for the reference regime
//   F.Correlation(pad_size=md, kernel_size=1, max_displacement=md, stride1=1, stride2=1, is_multiply=1) + LeakyReLU
//   network/MaskFlownet.py:193-195,217 (md=4) and :440-441,467 (md=2).
//
// These levels are small (1.7 .. 48 MB of algorithmic bytes, L2-resident in the network) and were latency / occupancy bound
// in round 1 (16..80 CTAs walking 2..7 channel chunks serially).  Here a CTA owns RB output rows x (8*TWB) pixels of one
// sample with ALL channels resident in shared memory, so an accumulator (row r, dy) is finished by one uninterrupted K loop
// and goes straight to the epilogue (no accumulators held across chunks, no inter-chunk barriers):
//   phase 1  all 8 warps: coalesced LDG (lane = pixel, 8 channel planes per unit) -> bf16 hi / lo split -> STS.128 into
//            pixel-major rows (pixel pitch = odd multiple of 16 B: conflict-free STS.128 and ldmatrix without swizzling);
//            data1 pre-scaled by 1/C; out-of-image positions and channels >= C are zeros (the operator's pad_size).
//   phase 2  warp = (8-pixel block, subset of the RB + 2 md data2 rows): per data2 row one ldmatrix sweep over K feeds the
//            mma.sync.m16n8k16 chains of every pixel row it serves (banded formulation: 16 data2 positions x 8 pixels -> all
//            dx of one dy; hi*lo + lo*hi + hi*hi, fp32 accumulate); LeakyReLU; per-warp staging; 32-byte plane-row stores.
// RB (4 / 2 / 1) and the strip width (32 / 16 pixels) are chosen by the host so that the grid covers all SMs.
#include <cuda_bf16.h>

#include "common.cuh"
#include "ptx.cuh"

namespace mfn {
namespace rb {
constexpr int NTHREADS = 256, NWARPS = 8, HX = 4;

// pixel pitch in bytes: 2 bytes x channels padded to 16, made an odd multiple of 16
__host__ __device__ inline int pixel_pitch(int C) {
  const int cp = (C + 15) / 16 * 16;
  return ((cp / 8) & 1) ? 2 * cp : 2 * cp + 16;
}
__host__ __device__ inline int smem_bytes(int C, int md, int rb_, int twb) {
  const int ps = pixel_pitch(C), tw = 8 * twb;
  return 2 * ((rb_ + 2 * md) * (tw + 2 * HX) + rb_ * tw) * ps + NWARPS * (2 * md + 1) * 8 * 4;
}
}  // namespace rb

template <int MD, int RB, int TWB>
__global__ void __launch_bounds__(rb::NTHREADS, 2)
    corr_rb_kernel(const float* __restrict__ d1, const float* __restrict__ d2, float* __restrict__ out, int C, int H, int W,
                   long long out_bs, float slope, int tilesX, int tilesY) {
  using namespace rb;
  constexpr int G = 2 * MD + 1, TW = 8 * TWB, NPOS = TW + 2 * HX, NROW = RB + 2 * MD;
  constexpr int NSEG2 = (NPOS + 31) / 32;
  extern __shared__ __align__(128) unsigned char smem[];
  const int PS = pixel_pitch(C), KS = (C + 15) / 16, CG = 2 * KS;
  const int F2_LO = NROW * NPOS * PS, F1_OFF = 2 * F2_LO, F1_LO = RB * TW * PS;
  unsigned char* f2s = smem;
  unsigned char* f1s = smem + F1_OFF;
  float* stg_all = reinterpret_cast<float*>(smem + F1_OFF + 2 * F1_LO);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tile = blockIdx.x;
  const int tx = tile % tilesX, ty = (tile / tilesX) % tilesY, n = tile / (tilesX * tilesY);
  const int x0 = tx * TW, y0 = ty * RB;
  const size_t plane = (size_t)H * W;
  const float invC = 1.f / (float)C;

  // ---------------- phase 1: load + split + transpose ----------------
  {
    const int U2 = NROW * NSEG2 * CG, U = U2 + RB * CG;
    const float* b1 = d1 + (size_t)n * C * plane;
    const float* b2 = d2 + (size_t)n * C * plane;
    constexpr int BATCH = 4;
    for (int u0 = warp * BATCH; u0 < U; u0 += NWARPS * BATCH) {
      float e[BATCH][8];
      unsigned char* dst[BATCH];
      int lo_off[BATCH];
      float sc[BATCH];
#pragma unroll
      for (int k = 0; k < BATCH; ++k) {
        const int u = u0 + k;
        dst[k] = nullptr;
        lo_off[k] = 0;
        sc[k] = 1.f;
        bool ok = false;
        const float* src = b2;
        int cg = 0;
        if (u < U) {
          cg = u % CG;
          const int v = u / CG;
          if (u < U2) {
            const int row = v / NSEG2, p = 32 * (v - row * NSEG2) + lane;
            const int y = y0 - MD + row, x = x0 - HX + p;
            if (p < NPOS) {
              dst[k] = f2s + (row * NPOS + p) * PS + cg * 16;
              lo_off[k] = F2_LO;
              ok = y >= 0 && y < H && x >= 0 && x < W;
              src = b2 + (size_t)y * W + x;
            }
          } else {
            const int row = v - NROW * NSEG2, p = lane;
            const int y = y0 + row, x = x0 + p;
            if (p < TW) {
              dst[k] = f1s + (row * TW + p) * PS + cg * 16;
              lo_off[k] = F1_LO;
              sc[k] = invC;
              ok = y < H && x < W;
              src = b1 + (size_t)y * W + x;
            }
          }
        }
        const int c0 = 8 * cg;
        src += (size_t)c0 * plane;
#pragma unroll
        for (int c = 0; c < 8; ++c) e[k][c] = (ok && c0 + c < C) ? __ldg(src + (size_t)c * plane) : 0.f;
      }
#pragma unroll
      for (int k = 0; k < BATCH; ++k) {
        if (dst[k]) {
          uint4 hi, lo;
          split_pair(e[k][0] * sc[k], e[k][1] * sc[k], hi.x, lo.x);
          split_pair(e[k][2] * sc[k], e[k][3] * sc[k], hi.y, lo.y);
          split_pair(e[k][4] * sc[k], e[k][5] * sc[k], hi.z, lo.z);
          split_pair(e[k][6] * sc[k], e[k][7] * sc[k], hi.w, lo.w);
          *reinterpret_cast<uint4*>(dst[k]) = hi;
          *reinterpret_cast<uint4*>(dst[k] + lo_off[k]) = lo;
        }
      }
    }
  }
  __syncthreads();

  // ---------------- phase 2: banded MMA + epilogue ----------------
  constexpr int NT = NWARPS / TWB;            // warps sharing one 8-pixel block: they interleave the data2 rows
  const int b = warp % TWB, tsub = warp / TWB;
  const int g = lane >> 2, j = lane & 3;
  const int l8 = lane & 7, mi = lane >> 3;
  const uint32_t f2_u32 = smem_u32(f2s), f1_u32 = smem_u32(f1s);
  const uint32_t offA = (uint32_t)((8 * b + 8 * (mi & 1) + l8) * PS + (mi >> 1) * 16);
  const uint32_t offB = (uint32_t)((8 * b + l8) * PS + (mi & 1) * 16 + (mi >> 1) * F1_LO);
  float* stg = stg_all + warp * (G * 8);
  int dxi[4];
  bool okv[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    dxi[i] = g + 8 * (i >> 1) - (2 * j + (i & 1)) - 4 + MD;
    okv[i] = dxi[i] >= 0 && dxi[i] < G;
  }
  float* obase = out + (size_t)n * out_bs;

  for (int t = tsub; t < NROW; t += NT) {
    float acc[RB][4];
#pragma unroll
    for (int r = 0; r < RB; ++r)
#pragma unroll
      for (int q = 0; q < 4; ++q) acc[r][q] = 0.f;
    const uint32_t arow = f2_u32 + (uint32_t)(t * NPOS * PS) + offA;
#pragma unroll 2
    for (int kk = 0; kk < KS; ++kk) {
      uint32_t ah[4], al[4];
      ldsm_x4(arow + (uint32_t)(kk * 32), ah);
      ldsm_x4(arow + (uint32_t)(kk * 32 + F2_LO), al);
#pragma unroll
      for (int r = 0; r < RB; ++r) {
        if (t - r < 0 || t - r >= G) continue;
        uint32_t bq[4];   // {hi k-half 0, hi k-half 1, lo k-half 0, lo k-half 1}
        ldsm_x4(f1_u32 + (uint32_t)(r * TW * PS + kk * 32) + offB, bq);
        mma_bf16(acc[r], ah, bq[2], bq[3]);
        mma_bf16(acc[r], al, bq[0], bq[1]);
        mma_bf16(acc[r], ah, bq[0], bq[1]);
      }
    }
#pragma unroll
    for (int r = 0; r < RB; ++r) {
      const int d = t - r;
      if (d < 0 || d >= G) continue;
#pragma unroll
      for (int i = 0; i < 4; ++i)
        if (okv[i]) stg[dxi[i] * 8 + 2 * j + (i & 1)] = leaky(acc[r][i], slope);
      __syncwarp();
      const int y = y0 + r;
      if (y < H) {
        float* orow = obase + ((size_t)(d * G) * H + y) * W + x0 + 8 * b;
        for (int e = lane; e < G * 8; e += 32) {
          const int dx = e >> 3, px = e & 7;
          if (x0 + 8 * b + px < W) orow[(size_t)dx * plane + px] = stg[e];
        }
      }
      __syncwarp();
    }
  }
}

template <int MD, int RB, int TWB>
static int launch_rb(const float* d1, const float* d2, float* out, int N, int C, int H, int W, long long obs, float slope,
                     cudaStream_t st) {
  using namespace rb;
  const int smem = smem_bytes(C, MD, RB, TWB);
  static SmemOptIn opt;
  {
    const cudaError_t e = ensure_dyn_smem(corr_rb_kernel<MD, RB, TWB>, smem, opt);
    if (e != cudaSuccess) return fail((int)e, "cudaFuncSetAttribute(corr_rb_kernel): %s", cudaGetErrorString(e));
  }
  const int tilesX = (W + 8 * TWB - 1) / (8 * TWB), tilesY = (H + RB - 1) / RB;
  const long long tiles = (long long)N * tilesX * tilesY;
  if (tiles >= (1LL << 31)) return -1;
  corr_rb_kernel<MD, RB, TWB><<<(unsigned)tiles, NTHREADS, smem, st>>>(d1, d2, out, C, H, W, obs, slope, tilesX, tilesY);
  static const char* names[6] = {"corr_rb_kernel<rb1,w32>", "corr_rb_kernel<rb2,w32>", "corr_rb_kernel<rb4,w32>",
                                 "corr_rb_kernel<rb1,w16>", "corr_rb_kernel<rb2,w16>", "corr_rb_kernel<rb4,w16>"};
  return check_launch(names[(RB == 1 ? 0 : (RB == 2 ? 1 : 2)) + (TWB == 2 ? 3 : 0)]);
}

// Returns -1 when no configuration fits the 227 KB of shared memory (caller falls back to the chunked tile kernel).
int launch_corr_rb(int md, const float* d1, const float* d2, float* out, int N, int C, int H, int W, long long obs, float slope,
                   cudaStream_t st) {
  using namespace rb;
  const int budget = 227 * 1024;
  // 16-pixel strips for narrow images (half the data2 positions): the smaller tile lets two CTAs share an SM, so one
  // CTA's load phase runs under the other's MMA phase
  const int twb = W <= 16 ? 2 : 4;
  const int tilesX = (W + 8 * twb - 1) / (8 * twb);
  int rbs = 4;
  auto ctas = [&](int r) { return (long long)N * tilesX * ((H + r - 1) / r); };
  while (rbs > 1 && (smem_bytes(C, md, rbs, twb) > budget || ctas(rbs) < kNumSMs)) rbs >>= 1;
  if (smem_bytes(C, md, rbs, twb) > budget) return -1;
#define MFN_RB(MD_, RB_, TWB_) launch_rb<MD_, RB_, TWB_>(d1, d2, out, N, C, H, W, obs, slope, st)
  if (md == 4) {
    if (twb == 4) return rbs == 4 ? MFN_RB(4, 4, 4) : (rbs == 2 ? MFN_RB(4, 2, 4) : MFN_RB(4, 1, 4));
    return rbs == 4 ? MFN_RB(4, 4, 2) : (rbs == 2 ? MFN_RB(4, 2, 2) : MFN_RB(4, 1, 2));
  }
  if (twb == 4) return rbs == 4 ? MFN_RB(2, 4, 4) : (rbs == 2 ? MFN_RB(2, 2, 4) : MFN_RB(2, 1, 4));
  return rbs == 4 ? MFN_RB(2, 4, 2) : (rbs == 2 ? MFN_RB(2, 2, 2) : MFN_RB(2, 1, 2));
#undef MFN_RB
}

}  // namespace mfn
