// corr_fwd.cu -- correlation cost-volume forward kernels (K1) for sm_90a.
//
// Serves mfn_correlation_forward (include/maskflow_b200.h), i.e. the reference's
//   F.Correlation(im1, im2, pad_size=md, kernel_size=1, max_displacement=md, stride1=1, stride2=1,
//                 is_multiply=1)        network/MaskFlownet.py:193-195 (md=4), :440-441 (md=2)
// followed by LeakyReLU(0.1) (:217 ...), fused as the epilogue.
//
// Three kernels:
//   corr_generic_kernel   every MXNet parameter combination, one thread per output element (exact fp32)
//   corr_simt_kernel      tiled fp32-FMA kernel for the reference regime (exact fp32 accumulation)
//   corr_mma_kernel       tensor-core kernel for the reference regime: operands split into bf16 hi/lo
//                         halves, 3 MMAs per product (hi*hi + hi*lo + lo*hi), fp32 accumulation.
//                         Warp-specialised: producer warps stream fp32 NCHW tiles from HBM/L2, split and
//                         transpose them into channel-contiguous bf16 tiles in shared memory; consumer warps
//                         run ldmatrix + mma.sync on a banded formulation (16 f2 positions x 8 pixels per
//                         MMA, 9/16 of the issued MACs useful) and write the D planes with coalesced stores.
#include <cuda_bf16.h>

#include "common.cuh"
#include "ptx.cuh"

namespace mfn {

// =====================================================================================================
// Generic kernel: literal MXNet semantics (zero padding handled by bounds tests instead of padded temps).
// =====================================================================================================
__global__ void corr_generic_kernel(const float* __restrict__ d1, const float* __restrict__ d2,
                                    float* __restrict__ out, int N, int C, int H, int W, int pad,
                                    int ks, int md, int s1, int s2, int is_mul, int D, int OH, int OW,
                                    long long out_bs, float slope) {
  const int G = 2 * (md / s2) + 1, r = md / s2;
  const long long total = (long long)N * D * OH * OW;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const int j = (int)(idx % OW);
    const int i = (int)((idx / OW) % OH);
    const int q = (int)((idx / ((long long)OW * OH)) % D);
    const int n = (int)(idx / ((long long)OW * OH * D));
    // coordinates in the UNPADDED inputs
    const int x1 = j * s1 + md - pad, y1 = i * s1 + md - pad;
    const int x2 = x1 + (q % G - r) * s2, y2 = y1 + (q / G - r) * s2;
    float acc = 0.f;
    for (int h = 0; h < ks; ++h)
      for (int w = 0; w < ks; ++w) {
        const int ya = y1 + h, xa = x1 + w, yb = y2 + h, xb = x2 + w;
        // outside the zero-padded extent nothing is read at all (MXNet's temporaries end there)
        if (ya < -pad || ya >= H + pad || xa < -pad || xa >= W + pad) continue;
        const bool ina = (ya >= 0 && ya < H && xa >= 0 && xa < W);
        const bool pb = (yb >= -pad && yb < H + pad && xb >= -pad && xb < W + pad);
        const bool inb = (yb >= 0 && yb < H && xb >= 0 && xb < W);
        if (is_mul) {
          if (!(ina && inb)) continue;
          const float* a = d1 + ((size_t)n * C * H + ya) * W + xa;
          const float* b = d2 + ((size_t)n * C * H + yb) * W + xb;
          for (int c = 0; c < C; ++c) acc += __ldg(a + (size_t)c * H * W) * __ldg(b + (size_t)c * H * W);
        } else {
          if (!pb) {  // d2 position beyond the padded temp: MXNet would read out of its buffer; we treat it as 0
            if (ina) {
              const float* a = d1 + ((size_t)n * C * H + ya) * W + xa;
              for (int c = 0; c < C; ++c) acc += fabsf(__ldg(a + (size_t)c * H * W));
            }
            continue;
          }
          for (int c = 0; c < C; ++c) {
            const float av = ina ? __ldg(d1 + (((size_t)n * C + c) * H + ya) * W + xa) : 0.f;
            const float bv = inb ? __ldg(d2 + (((size_t)n * C + c) * H + yb) * W + xb) : 0.f;
            acc += fabsf(av - bv);
          }
        }
      }
    const float v = acc / (float)(ks * ks * C);
    out[(size_t)n * out_bs + ((size_t)q * OH + i) * OW + j] = leaky(v, slope);
  }
}

// =====================================================================================================
// SIMT tiled kernel (exact fp32).  CTA tile = 8 rows x 32 pixels; thread = (dy, row, 4-pixel strip), holding
// 4 x G accumulators; channels staged in chunks of 16 through shared memory.
// =====================================================================================================
namespace simt {
constexpr int TH = 8, TW = 32, CK = 16;
}

template <int MD>
__global__ void __launch_bounds__(64 * (2 * MD + 1))
    corr_simt_kernel(const float* __restrict__ d1, const float* __restrict__ d2, float* __restrict__ out,
                     int N, int C, int H, int W, long long out_bs, float slope) {
  using namespace simt;
  constexpr int G = 2 * MD + 1;
  constexpr int HR = TH + 2 * MD;
  constexpr int HWD = TW + 8;  // f2 tile always carries a 4-pixel halo so that rows stay 16B aligned
  constexpr int NT = 64 * G;
  extern __shared__ __align__(16) float smem[];
  float* s1 = smem;                  // [CK][TH][TW]
  float* s2 = smem + CK * TH * TW;   // [CK][HR][HWD]

  const int tilesX = (W + TW - 1) / TW, tilesY = (H + TH - 1) / TH;
  const int tile = blockIdx.x;
  const int tx = tile % tilesX, ty = (tile / tilesX) % tilesY, n = tile / (tilesX * tilesY);
  const int x0 = tx * TW, y0 = ty * TH;
  const int tid = threadIdx.x;
  const int qx = tid & 7, r = (tid >> 3) & 7, dyi = tid >> 6;  // dyi in [0,G)

  float acc[G][4];
#pragma unroll
  for (int a = 0; a < G; ++a)
#pragma unroll
    for (int p = 0; p < 4; ++p) acc[a][p] = 0.f;

  const float* b1 = d1 + (size_t)n * C * H * W;
  const float* b2 = d2 + (size_t)n * C * H * W;
  for (int c0 = 0; c0 < C; c0 += CK) {
    __syncthreads();
    for (int e = tid; e < CK * TH * TW; e += NT) {
      const int xx = e % TW, yy = (e / TW) % TH, cc = e / (TW * TH);
      const int c = c0 + cc, y = y0 + yy, x = x0 + xx;
      s1[e] = (c < C && y < H && x < W) ? __ldg(b1 + ((size_t)c * H + y) * W + x) : 0.f;
    }
    for (int e = tid; e < CK * HR * HWD; e += NT) {
      const int xx = e % HWD, yy = (e / HWD) % HR, cc = e / (HWD * HR);
      const int c = c0 + cc, y = y0 - MD + yy, x = x0 - 4 + xx;
      s2[e] = (c < C && y >= 0 && y < H && x >= 0 && x < W) ? __ldg(b2 + ((size_t)c * H + y) * W + x) : 0.f;
    }
    __syncthreads();
#pragma unroll 4
    for (int cc = 0; cc < CK; ++cc) {
      const float4 a = *reinterpret_cast<const float4*>(s1 + (cc * TH + r) * TW + 4 * qx);
      const float* row = s2 + (cc * HR + r + dyi) * HWD + 4 * qx;  // element 0 == pixel x-4
      const float4 v0 = *reinterpret_cast<const float4*>(row);
      const float4 v1 = *reinterpret_cast<const float4*>(row + 4);
      const float4 v2 = *reinterpret_cast<const float4*>(row + 8);
      const float f[12] = {v0.x, v0.y, v0.z, v0.w, v1.x, v1.y, v1.z, v1.w, v2.x, v2.y, v2.z, v2.w};
      const float av[4] = {a.x, a.y, a.z, a.w};
#pragma unroll
      for (int dxi = 0; dxi < G; ++dxi)
#pragma unroll
        for (int p = 0; p < 4; ++p) acc[dxi][p] = fmaf(av[p], f[p + dxi + (4 - MD)], acc[dxi][p]);
    }
  }
  const int y = y0 + r, xb = x0 + 4 * qx;
  if (y >= H) return;
  const float inv = 1.f / (float)C;
  float* o = out + (size_t)n * out_bs + (size_t)y * W + xb;
  const bool vec = ((W & 3) == 0) && ((out_bs & 3) == 0) && ((reinterpret_cast<uintptr_t>(out) & 15) == 0);
#pragma unroll
  for (int dxi = 0; dxi < G; ++dxi) {
    float* op = o + (size_t)(dyi * G + dxi) * H * W;
    float v[4];
#pragma unroll
    for (int p = 0; p < 4; ++p) v[p] = leaky(acc[dxi][p] * inv, slope);
    if (vec && xb + 3 < W) {
      *reinterpret_cast<float4*>(op) = make_float4(v[0], v[1], v[2], v[3]);
    } else {
#pragma unroll
      for (int p = 0; p < 4; ++p)
        if (xb + p < W) op[p] = v[p];
    }
  }
}

// =====================================================================================================
// Tensor-core kernel (bf16 hi/lo split, mma.sync.m16n8k16).
// =====================================================================================================
namespace tc {
constexpr int TH = 4;    // tile rows
constexpr int TW = 32;   // tile pixels per row
constexpr int CK = 32;   // channels per pipeline stage
constexpr int RS = 2 * CK + 16;  // bytes per pixel row of a bf16 tile (80: odd multiple of 16 -> conflict-free ldmatrix)
constexpr int HX = 4;    // horizontal halo carried in shared memory (always 4 so that rows stay 16B aligned)
constexpr int HWP = TW + 2 * HX;  // 40 pixels per halo row
constexpr int NCONS = 8;          // consumer warps: (row 0..3) x (16-pixel half 0..1)
constexpr int NPROD = 8;          // producer warps (the profile of the 12 + 4 split showed the consumers waiting on them)
constexpr int NTHREADS = 32 * (NCONS + NPROD);
constexpr int OCT_PER_ROW = (TW + 16) / 8;  // aligned 8-pixel groups spanning [x0-8, x0+TW+8)
constexpr int STG_STRIDE = 20;    // floats per dx row of the per-warp output staging buffer

__host__ __device__ constexpr int halo_rows(int md) { return TH + 2 * md; }
__host__ __device__ constexpr int stage_bytes(int md) { return halo_rows(md) * HWP * RS * 2; }  // hi + lo
__host__ __device__ constexpr int smem_bytes(int md) {
  return 2 * stage_bytes(md) + NCONS * (2 * md + 1) * STG_STRIDE * 4 + 64;
}
}  // namespace tc

// VEC: rows are 16-byte aligned (W % 4 == 0 and 16B-aligned base) -> float4 producer loads.
template <int MD, bool VEC>
__global__ void __launch_bounds__(tc::NTHREADS, 1)
    corr_mma_kernel(const float* __restrict__ d1, const float* __restrict__ d2, float* __restrict__ out,
                    int N, int C, int H, int W, long long out_bs, float slope, int tilesX, int tilesY,
                    int numTiles) {
  using namespace tc;
  constexpr int G = 2 * MD + 1;
  constexpr int HR = halo_rows(MD);
  constexpr int STAGE = stage_bytes(MD);
  constexpr int LO_OFF = HR * HWP * RS;  // byte offset of the "lo" tile inside a stage

  extern __shared__ __align__(128) unsigned char smem_raw[];
  unsigned char* stage0 = smem_raw;
  float* stg_all = reinterpret_cast<float*>(smem_raw + 2 * STAGE);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem_raw + 2 * STAGE + NCONS * G * STG_STRIDE * 4);
  const uint32_t bar_full = smem_u32(bars);        // [2]
  const uint32_t bar_empty = smem_u32(bars + 2);   // [2]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    mbar_init(bar_full, NPROD * 32);
    mbar_init(bar_full + 8, NPROD * 32);
    mbar_init(bar_empty, NCONS);
    mbar_init(bar_empty + 8, NCONS);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  const int nChunks = (C + CK - 1) / CK;
  const size_t plane = (size_t)H * W;

  if (warp >= NCONS) {
    // ================================ PRODUCERS ================================
    const int pw = warp - NCONS;
    const int m = lane >> 4;   // which aligned quad of the octet
    const int j = lane & 15;   // channel pair inside the chunk
    uint32_t s = 0;
    for (int tile = blockIdx.x; tile < numTiles; tile += gridDim.x) {
      const int tx = tile % tilesX, ty = (tile / tilesX) % tilesY, n = tile / (tilesX * tilesY);
      const int x0 = tx * TW, y0 = ty * TH;
      const float* base = d2 + (size_t)n * C * plane;
      for (int ch = 0; ch < nChunks; ++ch, ++s) {
        const uint32_t b = s & 1u, u = s >> 1;
        mbar_wait(bar_empty + 8 * b, (u & 1u) ^ 1u);
        unsigned char* st = stage0 + b * STAGE;
        const int ca = ch * CK + 2 * j;
        const bool c_ok0 = ca < C, c_ok1 = ca + 1 < C;
        const float* pc = base + (size_t)ca * plane;
        constexpr int NOR = HR * OCT_PER_ROW;  // octet-rows in this stage
        constexpr int U = 5;  // 10 independent 16-byte loads per thread in flight
        for (int o0 = pw; o0 < NOR; o0 += NPROD * U) {
          float4 v0[U], v1[U];
          int pxr[U], rr[U];
#pragma unroll
          for (int uu = 0; uu < U; ++uu) {
            const int o = o0 + uu * NPROD;
            v0[uu] = make_float4(0.f, 0.f, 0.f, 0.f);
            v1[uu] = v0[uu];
            rr[uu] = o / OCT_PER_ROW;
            const int oct = o - rr[uu] * OCT_PER_ROW;
            pxr[uu] = 8 * oct + 4 * m - HX;  // pixel index inside the halo row; -4 and 40 are the masked quads
            const int y = y0 - MD + rr[uu];
            const int x = x0 - 8 + 8 * oct + 4 * m;
            if (o < NOR && pxr[uu] >= 0 && pxr[uu] < HWP && y >= 0 && y < H) {
              const float* p = pc + (size_t)y * W + x;
              if (VEC) {
                if (x >= 0 && x < W) {  // W % 4 == 0: the quad is entirely inside or outside
                  if (c_ok0) v0[uu] = __ldg(reinterpret_cast<const float4*>(p));
                  if (c_ok1) v1[uu] = __ldg(reinterpret_cast<const float4*>(p + plane));
                }
              } else {
                float t0[4] = {0.f, 0.f, 0.f, 0.f}, t1[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
                for (int e = 0; e < 4; ++e)
                  if (x + e >= 0 && x + e < W) {
                    if (c_ok0) t0[e] = __ldg(p + e);
                    if (c_ok1) t1[e] = __ldg(p + plane + e);
                  }
                v0[uu] = make_float4(t0[0], t0[1], t0[2], t0[3]);
                v1[uu] = make_float4(t1[0], t1[1], t1[2], t1[3]);
              }
            }
          }
#pragma unroll
          for (int uu = 0; uu < U; ++uu) {
            const int o = o0 + uu * NPROD;
            if (o < NOR && pxr[uu] >= 0 && pxr[uu] < HWP) {
              unsigned char* dst = st + (size_t)(rr[uu] * HWP + pxr[uu]) * RS + 4 * j;
              const float a[4] = {v0[uu].x, v0[uu].y, v0[uu].z, v0[uu].w};
              const float c[4] = {v1[uu].x, v1[uu].y, v1[uu].z, v1[uu].w};
#pragma unroll
              for (int e = 0; e < 4; ++e) {
                uint32_t hi, lo;
                split_pair(a[e], c[e], hi, lo);
                *reinterpret_cast<uint32_t*>(dst + e * RS) = hi;
                *reinterpret_cast<uint32_t*>(dst + e * RS + LO_OFF) = lo;
              }
            }
          }
        }
        mbar_arrive(bar_full + 8 * b);  // release: this thread's tile writes are visible to waiters
      }
    }
  } else {
    // ================================ CONSUMERS ================================
    const int r = warp >> 1;            // tile row of this warp's item
    const int xs = (warp & 1) * 16;     // first pixel (tile-relative) of the 16-pixel item
    const int g = lane >> 2, j = lane & 3;
    float* stg = stg_all + warp * (G * STG_STRIDE);
    const float invC = 1.f / (float)C;

    // per-lane ldmatrix byte offsets inside a stage (excluding the dy row and k-step terms)
    const int l8 = lane & 7, mi = lane >> 3;
    // loads 1/2: matrices (block mi&1, k-half mi>>1) of the hi / lo tile
    const uint32_t off12 = (uint32_t)((xs + 8 * (mi & 1) + l8) * RS + 16 * (mi >> 1));
    // load 3: matrices (hi|lo = mi>>1, block 2, k-half mi&1)
    const uint32_t off3 = (uint32_t)((xs + 16 + l8) * RS + 16 * (mi & 1) + (mi >> 1) * LO_OFF);

    uint32_t s = 0;
    for (int tile = blockIdx.x; tile < numTiles; tile += gridDim.x) {
      const int tx = tile % tilesX, ty = (tile / tilesX) % tilesY, n = tile / (tilesX * tilesY);
      const int x0 = tx * TW, y0 = ty * TH;
      const int y = y0 + r;
      const float* f1n = d1 + (size_t)n * C * plane;

      float acc[G][2][4];
#pragma unroll
      for (int d = 0; d < G; ++d)
#pragma unroll
        for (int t = 0; t < 2; ++t)
#pragma unroll
          for (int i = 0; i < 4; ++i) acc[d][t][i] = 0.f;

      for (int ch = 0; ch < nChunks; ++ch, ++s) {
        const uint32_t b = s & 1u, u = s >> 1;
        // ---- B fragments (data1) straight from global memory: lane (g, j) owns pixel g, channels 2j.. ----
        uint32_t bh[2][2][2], bl[2][2][2];  // [k-step][tile][reg]
#pragma unroll
        for (int kk = 0; kk < 2; ++kk)
#pragma unroll
          for (int t = 0; t < 2; ++t) {
            const int x = x0 + xs + 8 * t + g;
            const int c = ch * CK + 16 * kk + 2 * j;
            const bool ok = (y < H) && (x < W);
            const float* p = f1n + (size_t)c * plane + (size_t)y * W + x;
            const float e0 = (ok && c < C) ? __ldg(p) : 0.f;
            const float e1 = (ok && c + 1 < C) ? __ldg(p + plane) : 0.f;
            const float e8 = (ok && c + 8 < C) ? __ldg(p + 8 * plane) : 0.f;
            const float e9 = (ok && c + 9 < C) ? __ldg(p + 9 * plane) : 0.f;
            split_pair(e0, e1, bh[kk][t][0], bl[kk][t][0]);
            split_pair(e8, e9, bh[kk][t][1], bl[kk][t][1]);
          }
        mbar_wait(bar_full + 8 * b, u & 1u);
        const uint32_t st = smem_u32(stage0 + b * STAGE);
#pragma unroll
        for (int kk = 0; kk < 2; ++kk) {
#pragma unroll
          for (int d = 0; d < G; ++d) {
            const uint32_t rowoff = (uint32_t)((r + d) * HWP * RS + 32 * kk);
            uint32_t h[4], l[4], x3[4];
            ldsm_x4(st + rowoff + off12, h);
            ldsm_x4(st + rowoff + off12 + LO_OFF, l);
            ldsm_x4(st + rowoff + off3, x3);
            // tile 0: rows = blocks 0,1 ; tile 1: rows = blocks 1,2
            const uint32_t h1[4] = {h[1], x3[0], h[3], x3[1]}, l1[4] = {l[1], x3[2], l[3], x3[3]};
            mma_bf16(acc[d][0], h, bl[kk][0][0], bl[kk][0][1]);
            mma_bf16(acc[d][0], l, bh[kk][0][0], bh[kk][0][1]);
            mma_bf16(acc[d][0], h, bh[kk][0][0], bh[kk][0][1]);
            mma_bf16(acc[d][1], h1, bl[kk][1][0], bl[kk][1][1]);
            mma_bf16(acc[d][1], l1, bh[kk][1][0], bh[kk][1][1]);
            mma_bf16(acc[d][1], h1, bh[kk][1][0], bh[kk][1][1]);
          }
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(bar_empty + 8 * b);
      }

      // ---- epilogue: accumulators -> per-warp staging -> coalesced plane rows ----
      // accumulator (row, col) of tile t: f2 position xs+8t-4+row versus pixel xs+8t+col  =>  dx = row-col-4
      float* obase = out + (size_t)n * out_bs + (size_t)y * W + (x0 + xs);
      const int p = lane & 15, hsel = lane >> 4;
#pragma unroll
      for (int d = 0; d < G; ++d) {
#pragma unroll
        for (int t = 0; t < 2; ++t)
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const int row = g + 8 * (i >> 1), col = 2 * j + (i & 1);
            const int dxi = row - col - 4 + MD;
            if (dxi >= 0 && dxi < G) stg[dxi * STG_STRIDE + 8 * t + col] = leaky(acc[d][t][i] * invC, slope);
          }
        __syncwarp();
        if (y < H && x0 + xs + p < W) {
#pragma unroll
          for (int dxi = hsel; dxi < G; dxi += 2)
            obase[(size_t)(d * G + dxi) * plane + p] = stg[dxi * STG_STRIDE + p];
        }
        __syncwarp();
      }
    }
  }
}

// =====================================================================================================
// Tensor-core kernel, strip-marching variant for C <= 32 (one channel chunk): the dominant levels (v4).
//
// A CTA (16 symmetric warps, persistent, one per SM) owns a contiguous run of 8x32-pixel tiles in (n, x-strip, y) order
// and marches down each strip.  Shared memory holds, in split-bf16 (hi | lo), pixel-major form with 64 B per pixel and
// XOR-swizzled 16-byte chunks (conflict-free ldmatrix and STS without padding):
//   * a ring of 24 data2 rows: the 16 halo rows of the current tile + the 8 new rows of the next one (a tile that
//     continues a strip loads only its 8 new rows),
//   * two stages of 8 data1 rows (pre-scaled by 1/C).
// Software pipeline per tile, identical in every warp:
//   1. fire-and-forget `prefetch.global.L2` of the NEXT tile's 128-byte lines (no registers, no scoreboard: the DRAM reads
//      run under the tensor work; a register prefetch here was measured NOT to overlap with the MMAs)
//   2. current tile: B fragments (data1) by ldmatrix; walk the halo rows: each ldmatrix'ed A row (16 data2 positions x
//      16 channels, hi and lo) feeds the MMAs of both pixel rows of the warp's item (2 rows x 8 pixels): hi*lo + lo*hi +
//      hi*hi into fp32 accumulators; dy in passes of 3.  Per pass the four warps of a row pair drop their band pieces
//      (predicated STS, lane-constant predicates) into a shared [plane][32 px] staging buffer and then store full
//      128-byte plane rows (16-byte LDS, LeakyReLU, 16-byte STG: 4 lines per store instruction).
//      Before the last pass the next tile's rows are pulled from L2 into registers: lane = pixel, 8 channels per load
//      unit, every LDG covers whole sectors of 1-4 lines (2 data1 units + 2 data2 units + 1 halo-column unit per warp).
//   3. split / transpose those registers into the ring and the other data1 stage (one STS.128 per 8 channels)
//   4. __syncthreads
// Work assignment: each (n, x-strip) column of tiles is cut into equal pieces, one CTA per piece (level 2 of BASELINE
// configs[1]: 64 strips x 2 pieces of 7 tiles = 128 CTAs), so only the first tile of a CTA loads its full halo.
// =====================================================================================================
namespace r4 {
constexpr int TH = 8, TW = 32, HX = 4, HWP = TW + 2 * HX;
constexpr int NTHREADS = 64 * TH;                // 16 warps
constexpr int PXB = 64;                          // bytes per pixel (32 channels bf16), no padding
constexpr int ROW_BYTES = HWP * PXB;             // 2560: one split row (hi or lo)
constexpr int F1_ROW_BYTES = TW * PXB;           // 2048
constexpr int PASS = 3;
constexpr int SSTR = TW + 4;                     // staging row: the tile's 32 pixels + 4 pad (keeps float4 alignment)
constexpr int UPW = 5;                           // units per warp per batch: 4*TH + 6*TH = 10*TH = 2*TH warps x 5
constexpr int RING_ROWS = 2 * TH + 8;            // halo rows of a tile (md = 4) + TH new rows
__host__ __device__ constexpr int stg_group_bytes(int md) { return 2 * PASS * (2 * md + 1) * SSTR * 4; }  // 2 buffers
__host__ __device__ constexpr int smem_bytes(int md) {
  return 2 * RING_ROWS * ROW_BYTES + 2 * 2 * TH * F1_ROW_BYTES + (TH / 2) * stg_group_bytes(md);
}
}  // namespace r4

template <int MD, bool VEC>
__global__ void __launch_bounds__(r4::NTHREADS, 1)
    corr_mma_ring_kernel(const float* __restrict__ d1, const float* __restrict__ d2, float* __restrict__ out,
                         int N, int C, int H, int W, long long out_bs, float slope, int tilesX, int tilesY,
                         int numTiles, int ovec) {
  using namespace r4;
  constexpr int NWARPS = 2 * TH;
  constexpr int R = RING_ROWS, RING_LO = R * ROW_BYTES, RING_BYTES = 2 * RING_LO;
  constexpr int F1_LO = TH * F1_ROW_BYTES, F1_STAGE = 2 * F1_LO;
  constexpr int UNITS_F1 = TH * 4;                 // load units (32 lanes x 8 channels) of the data1 rows
  static_assert(UNITS_F1 + 6 * TH == UPW * NWARPS, "unit split of a continuing tile must be exact");
  constexpr int G = 2 * MD + 1;
  constexpr int HR = TH + 2 * MD;
  constexpr int NPASS = (G + PASS - 1) / PASS;
  constexpr int SROWS = PASS * G;   // staging rows (= output planes) per pass

  extern __shared__ __align__(128) unsigned char smem_raw[];
  unsigned char* ring = smem_raw;
  unsigned char* f1s = smem_raw + RING_BYTES;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // work assignment: a CTA owns one contiguous piece of one (n, x-strip) column of tiles -- numTiles here is the number
  // of pieces per strip; strips are never changed mid-run, so only the prologue tile is "fresh"
  const int ppS = numTiles;
  const int strip = blockIdx.x / ppS, piece = blockIdx.x - strip * ppS;
  const int ty_begin = (tilesY * piece) / ppS, ty_end = (tilesY * (piece + 1)) / ppS;
  const int t_begin = strip * tilesY + ty_begin;
  const int nStages = ty_end - ty_begin;
  const size_t plane = (size_t)H * W;
  const float invC = 1.f / (float)C;

  struct TileGeo {
    int n, x0, y0, first_slot, rr0, nrows;  // nrows = data2 halo rows to load (8 continuing, HR fresh), starting at rr0
    bool fresh;
  };
  auto geo = [&](int s, int& wr) {
    TileGeo t;
    const int tile = t_begin + s;
    const int ty = tile % tilesY, tx = (tile / tilesY) % tilesX;
    t.n = tile / (tilesY * tilesX);
    t.x0 = tx * TW;
    t.y0 = ty * TH;
    t.fresh = (s == 0);
    (void)ty;
    t.first_slot = t.fresh ? wr : (wr + R - 2 * MD) % R;
    t.rr0 = t.fresh ? 0 : 2 * MD;
    t.nrows = t.fresh ? HR : TH;
    wr = (wr + t.nrows) % R;
    return t;
  };
  // ---- load units: 32 lanes x 8 channels of one 16-byte smem chunk per pixel; every LDG touches full sectors of 1-4 lines.
  //   ids [0, 32)                     data1 row id>>2, pixels x0..x0+31 (one 128-byte line per channel), chunk id&3
  //   ids [32, 32+4*nrows)            data2 halo row (k>>2), pixels x0..x0+31, chunk k&3
  //   ids [.., .. + 2*nrows)          data2 halo columns: 2 rows x (left octet | right octet), chunk k&3
  struct UnitPos {
    bool is1, active;  // data1 unit? / does this lane carry a pixel that is stored
    int row;           // data1 tile row or data2 halo row
    int chunk, pidx;   // 16-byte chunk (8 channels); pixel index inside the smem row
    int y, x;          // image coordinates
  };
  auto unit_pos = [&](const TileGeo& t, int id) {
    UnitPos u;
    const int nmain = 4 * t.nrows;
    u.active = id < UNITS_F1 + nmain + 2 * t.nrows;
    u.is1 = id < UNITS_F1;
    if (u.is1) {
      u.row = id >> 2;
      u.chunk = id & 3;
      u.pidx = lane;
      u.y = t.y0 + u.row;
      u.x = t.x0 + lane;
    } else if (id < UNITS_F1 + nmain) {
      const int k = id - UNITS_F1;
      u.row = t.rr0 + (k >> 2);
      u.chunk = k & 3;
      u.pidx = HX + lane;
      u.y = t.y0 - MD + u.row;
      u.x = t.x0 + lane;
    } else {
      const int k = id - UNITS_F1 - nmain;
      const int blk = lane >> 3, px8 = lane & 7, side = blk & 1;
      u.row = t.rr0 + 2 * (k >> 2) + (blk >> 1);
      u.chunk = k & 3;
      u.pidx = side ? TW + HX + px8 : px8 - HX;
      u.x = side ? t.x0 + TW + px8 : t.x0 - 8 + px8;
      u.y = t.y0 - MD + u.row;
      u.active = u.active && (side ? px8 < HX : px8 >= HX);
    }
    return u;
  };
  auto load_unit = [&](const TileGeo& t, int id, float (&e)[8]) {
    const UnitPos u = unit_pos(t, id);
    const bool ok = u.active && u.y >= 0 && u.y < H && u.x >= 0 && u.x < W;
    const int c0 = 8 * u.chunk;
    const float* p = (u.is1 ? d1 : d2) + ((size_t)t.n * C + c0) * plane + (size_t)u.y * W + u.x;
#pragma unroll
    for (int c = 0; c < 8; ++c) e[c] = (ok && c0 + c < C) ? __ldg(p + (size_t)c * plane) : 0.f;
  };
  auto store_unit = [&](const TileGeo& t, int id, int f1stage, const float (&e)[8]) {
    const UnitPos u = unit_pos(t, id);
    if (!u.active) return;
    unsigned char* rowp;
    int lo_off;
    float sc;
    if (u.is1) {
      rowp = f1s + f1stage * F1_STAGE + u.row * F1_ROW_BYTES;
      lo_off = F1_LO;
      sc = invC;
    } else {
      int slot = t.first_slot + u.row;
      slot = slot >= 2 * R ? slot - 2 * R : (slot >= R ? slot - R : slot);
      rowp = ring + slot * ROW_BYTES;
      lo_off = RING_LO;
      sc = 1.f;
    }
    uint4 hi, lo;
    split_pair(e[0] * sc, e[1] * sc, hi.x, lo.x);
    split_pair(e[2] * sc, e[3] * sc, hi.y, lo.y);
    split_pair(e[4] * sc, e[5] * sc, hi.z, lo.z);
    split_pair(e[6] * sc, e[7] * sc, hi.w, lo.w);
    unsigned char* dst = rowp + swz(u.pidx, u.chunk);
    *reinterpret_cast<uint4*>(dst) = hi;
    *reinterpret_cast<uint4*>(dst + lo_off) = lo;
  };

  // ---- consumer-side lane constants: item = pixel rows 2rp, 2rp+1 x pixels 8oc..8oc+7 of the tile ----
  const int rp = warp >> 2, oc = warp & 3;
  const int g = lane >> 2, j = lane & 3;
  const int l8 = lane & 7, mi = lane >> 3;
  const int sw = (l8 >> 1) & 3;   // swizzle term of this lane's ldmatrix rows (pixel index = multiple of 8 + l8)
  const uint32_t ring_u32 = smem_u32(ring), f1_u32 = smem_u32(f1s);
  // A (ring): matrices (8-row block mi&1, k-half mi>>1) -> a0..a3;  B (data1 stage): matrices (hi|lo = mi>>1, k-half mi&1)
  uint32_t offA[2], offB[2];
#pragma unroll
  for (int kk = 0; kk < 2; ++kk) {
    offA[kk] = (uint32_t)((8 * oc + 8 * (mi & 1) + l8) * PXB + (((2 * kk + (mi >> 1)) ^ sw) << 4));
    offB[kk] = (uint32_t)((8 * oc + l8) * PXB + (((2 * kk + (mi & 1)) ^ sw) << 4) + (mi >> 1) * F1_LO);
  }
  // accumulator element i of this lane: (row, col) = (g + 8*(i>>1), 2j + (i&1));  dx index = row - col - 4 + MD
  bool okv[4];
  int sto[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int dxi = g + 8 * (i >> 1) - 2 * j - (i & 1) - 4 + MD;
    okv[i] = dxi >= 0 && dxi < G;
    sto[i] = dxi * SSTR + 8 * oc + 2 * j + (i & 1);
  }
  // the four warps of a row pair share a staging area (two buffers: one per pixel row) and a named barrier
  float* stg_g = reinterpret_cast<float*>(smem_raw + RING_BYTES + 2 * F1_STAGE) + rp * (2 * SROWS * SSTR);
  const int tig = threadIdx.x & 127;  // thread index inside the row-pair group
  auto group_sync = [&]() { asm volatile("bar.sync %0, 128;" ::"r"(1 + rp) : "memory"); };

  // ---- steady-state load roles (a continuing tile = 80 units): every warp takes two data1 units (row w>>1, 16 channels),
  //      two data2 units (new row w>>1, 16 channels) and one halo-column unit (row pair w>>2, chunk w&3): addresses are a
  //      base pointer + k*plane, shared-memory offsets are lane constants ----
  const int lr = warp >> 1, lc = 2 * (warp & 1);
  const int hrp2 = 2 * (warp >> 2), hch = warp & 3;
  const int hblk = lane >> 3, hpx8 = lane & 7, hside = hblk & 1;
  const bool hact = hside ? hpx8 < HX : hpx8 >= HX;
  const int hdx = hside ? TW + hpx8 : hpx8 - 8;
  const int hrow = 2 * MD + hrp2 + (hblk >> 1);                 // halo row of this lane's halo-column pixel
  const uint32_t so_f1a = (uint32_t)(lr * F1_ROW_BYTES + swz(lane, lc)), so_f1b = (uint32_t)(lr * F1_ROW_BYTES + swz(lane, lc + 1));
  const uint32_t so_ma = (uint32_t)swz(HX + lane, lc), so_mb = (uint32_t)swz(HX + lane, lc + 1);
  const uint32_t so_h = (uint32_t)swz(hside ? TW + HX + hpx8 : hpx8 - HX, hch);
  const bool fullC = (C == 32);      // no per-channel predicates needed
  const size_t plane4 = plane;       // element stride between channel planes
  auto prefetch_next = [&](const TileGeo& t, float (&e1)[16], float (&e2)[16], float (&eh)[8]) {
    // running pointers (p += plane) instead of per-load 64-bit multiplies
    const size_t nbase = (size_t)t.n * C;
    {
      const int y = t.y0 + lr, x = t.x0 + lane;
      const bool ok = y < H && x < W;
      const float* p = d1 + (nbase + 8 * lc) * plane + (size_t)y * W + x;
      if (fullC) {
        if (ok) {
#pragma unroll
          for (int c = 0; c < 16; ++c) { e1[c] = __ldg(p); p += plane4; }
        } else {
#pragma unroll
          for (int c = 0; c < 16; ++c) e1[c] = 0.f;
        }
      } else {
#pragma unroll
        for (int c = 0; c < 16; ++c) { e1[c] = (ok && 8 * lc + c < C) ? __ldg(p) : 0.f; p += plane4; }
      }
    }
    {
      const int y = t.y0 + MD + lr, x = t.x0 + lane;   // halo row 2*MD + lr
      const bool ok = y < H && x < W;
      const float* p = d2 + (nbase + 8 * lc) * plane + (size_t)y * W + x;
      if (fullC) {
        if (ok) {
#pragma unroll
          for (int c = 0; c < 16; ++c) { e2[c] = __ldg(p); p += plane4; }
        } else {
#pragma unroll
          for (int c = 0; c < 16; ++c) e2[c] = 0.f;
        }
      } else {
#pragma unroll
        for (int c = 0; c < 16; ++c) { e2[c] = (ok && 8 * lc + c < C) ? __ldg(p) : 0.f; p += plane4; }
      }
    }
    {
      const int y = t.y0 - MD + hrow, x = t.x0 + hdx;
      const bool ok = hact && y < H && x >= 0 && x < W;
      const float* p = d2 + (nbase + 8 * hch) * plane + (size_t)y * W + x;
      if (fullC) {
        if (ok) {
#pragma unroll
          for (int c = 0; c < 8; ++c) { eh[c] = __ldg(p); p += plane4; }
        } else {
#pragma unroll
          for (int c = 0; c < 8; ++c) eh[c] = 0.f;
        }
      } else {
#pragma unroll
        for (int c = 0; c < 8; ++c) { eh[c] = (ok && 8 * hch + c < C) ? __ldg(p) : 0.f; p += plane4; }
      }
    }
  };
  auto put_chunk = [&](unsigned char* dst, int lo_off, const float* e, float sc) {
    uint4 hi, lo;
    split_pair(e[0] * sc, e[1] * sc, hi.x, lo.x);
    split_pair(e[2] * sc, e[3] * sc, hi.y, lo.y);
    split_pair(e[4] * sc, e[5] * sc, hi.z, lo.z);
    split_pair(e[6] * sc, e[7] * sc, hi.w, lo.w);
    *reinterpret_cast<uint4*>(dst) = hi;
    *reinterpret_cast<uint4*>(dst + lo_off) = lo;
  };
  auto store_next = [&](const TileGeo& t, int f1stage, const float (&e1)[16], const float (&e2)[16], const float (&eh)[8]) {
    unsigned char* f1p = f1s + f1stage * F1_STAGE;
    put_chunk(f1p + so_f1a, F1_LO, &e1[0], invC);
    put_chunk(f1p + so_f1b, F1_LO, &e1[8], invC);
    int slot = t.first_slot + 2 * MD + lr;
    slot = slot >= 2 * R ? slot - 2 * R : (slot >= R ? slot - R : slot);
    unsigned char* rp2 = ring + slot * ROW_BYTES;
    put_chunk(rp2 + so_ma, RING_LO, &e2[0], 1.f);
    put_chunk(rp2 + so_mb, RING_LO, &e2[8], 1.f);
    if (hact) {
      int hs = t.first_slot + hrow;
      hs = hs >= 2 * R ? hs - 2 * R : (hs >= R ? hs - R : hs);
      put_chunk(ring + hs * ROW_BYTES + so_h, RING_LO, &eh[0], 1.f);
    }
  };

  // fire-and-forget L2 prefetch of a continuing tile's lines (one 128-byte line per (row, channel)): threads 0..255 take
  // the data1 rows, 256..511 the new data2 rows.  No register, no scoreboard: DRAM reads overlap the tensor work, and the
  // register loads at the end of the current tile hit L2.
  auto l2_prefetch_tile = [&](const TileGeo& t) {
    const int tt = threadIdx.x % (NTHREADS / 2), row = tt >> 5, ch = tt & 31;
    const bool second = threadIdx.x >= NTHREADS / 2;
    const int y = second ? t.y0 + MD + row : t.y0 + row;
    if (ch < C && y < H) {
      const float* p = (second ? d2 : d1) + ((size_t)t.n * C + ch) * plane + (size_t)y * W + t.x0;
      asm volatile("prefetch.global.L2 [%0];" ::"l"(p));
    }
  };

  // ---- prologue: bring in tile 0 completely ----
  int wr = 0;
  TileGeo cur = geo(0, wr);
  {
    constexpr int UALL = UNITS_F1 + 6 * HR;               // units of a fresh tile
    constexpr int UB = 8;                                 // units per warp per batch of loads (registers: 8 floats each)
    constexpr int NB = (UALL + UB * NWARPS - 1) / (UB * NWARPS);
#pragma unroll 1
    for (int b = 0; b < NB; ++b) {
      float e[UB][8];
      const int u0 = (b * NWARPS + warp) * UB;
#pragma unroll
      for (int k = 0; k < UB; ++k) load_unit(cur, u0 + k, e[k]);
#pragma unroll
      for (int k = 0; k < UB; ++k) store_unit(cur, u0 + k, 0, e[k]);
    }
  }
  __syncthreads();

  for (int s = 0; s < nStages; ++s) {
    // ---- 1. L2-prefetch the next tile's rows ----
    const bool has_next = s + 1 < nStages;
    TileGeo nxt = cur;
    float pe1[16], pe2[16], peh[8];
    if (has_next) {
      nxt = geo(s + 1, wr);   // always a continuing tile: its 8 new rows go to the 8 ring slots the current tile does not use
      l2_prefetch_tile(nxt);
    }

    // ---- 2. current tile ----
    uint32_t bq[2][2][4];   // [pixel row][kk] -> {hi k-half 0, hi k-half 1, lo k-half 0, lo k-half 1}
#pragma unroll
    for (int rw = 0; rw < 2; ++rw)
#pragma unroll
      for (int kk = 0; kk < 2; ++kk)
        ldsm_x4(f1_u32 + (uint32_t)((s & 1) * F1_STAGE + (2 * rp + rw) * F1_ROW_BYTES) + offB[kk], bq[rw][kk]);
    const int yA = cur.y0 + 2 * rp;
    float* obase = out + (size_t)cur.n * out_bs + (size_t)yA * W + cur.x0;
    const bool two_k = C > 16;

#pragma unroll
    for (int ps = 0; ps < NPASS; ++ps) {
      const int d0 = ps * PASS;
      // the next tile's lines were L2-prefetched at tile start: pull them into registers one pass before they are needed
      // (short L2-hit latency, hidden behind the last pass)
      if (ps == NPASS - 1 && has_next) prefetch_next(nxt, pe1, pe2, peh);
      float acc[2][PASS][4];
#pragma unroll
      for (int rw = 0; rw < 2; ++rw)
#pragma unroll
        for (int dd = 0; dd < PASS; ++dd)
#pragma unroll
          for (int i = 0; i < 4; ++i) acc[rw][dd][i] = 0.f;
      {
        // flat list of (kk, hh) steps; the fragments of step i+1 are fetched before the MMAs of step i are issued
        constexpr int NST = 2 * (PASS + 1);
        uint32_t ah[2][4], al[2][4];
        auto frag = [&](int st, uint32_t (&fh)[4], uint32_t (&fl)[4]) {
          const int kk = st / (PASS + 1), hh = st % (PASS + 1);
          int slot = cur.first_slot + 2 * rp + d0 + hh;
          slot = slot >= 2 * R ? slot - 2 * R : (slot >= R ? slot - R : slot);
          const uint32_t rowoff = ring_u32 + (uint32_t)(slot * ROW_BYTES) + offA[kk];
          ldsm_x4(rowoff, fh);
          ldsm_x4(rowoff + RING_LO, fl);
        };
        frag(0, ah[0], al[0]);
#pragma unroll
        for (int st = 0; st < NST; ++st) {
          const int kk = st / (PASS + 1), hh = st % (PASS + 1);
          if (kk == 1 && !two_k) break;
          if (st + 1 < NST) frag(st + 1, ah[(st + 1) & 1], al[(st + 1) & 1]);
          // halo row 2rp + d0 + hh serves (pixel row 0, dd = hh) and (pixel row 1, dd = hh-1)
          const bool useA = hh < PASS && d0 + hh < G;
          const bool useB = hh >= 1 && d0 + hh - 1 < G;
          uint32_t(&fh)[4] = ah[st & 1];
          uint32_t(&fl)[4] = al[st & 1];
          if (useA) {
            float(&a)[4] = acc[0][hh < PASS ? hh : 0];
            mma_bf16(a, fh, bq[0][kk][2], bq[0][kk][3]);
            mma_bf16(a, fl, bq[0][kk][0], bq[0][kk][1]);
            mma_bf16(a, fh, bq[0][kk][0], bq[0][kk][1]);
          }
          if (useB) {
            float(&a)[4] = acc[1][hh >= 1 ? hh - 1 : 0];
            mma_bf16(a, fh, bq[1][kk][2], bq[1][kk][3]);
            mma_bf16(a, fl, bq[1][kk][0], bq[1][kk][1]);
            mma_bf16(a, fh, bq[1][kk][0], bq[1][kk][1]);
          }
        }
      }
      // ---- epilogue of this pass (cooperative across the 4 warps of the row pair): each warp drops its 8-pixel band
      //      pieces into the group's [plane][32 px] staging buffer; then the 128 threads store full 128-byte plane rows ----
      const int nrow = (G - d0 < PASS ? G - d0 : PASS) * G;   // planes of this pass
#pragma unroll
      for (int rw = 0; rw < 2; ++rw) {
        float* sb = stg_g + rw * (SROWS * SSTR);
#pragma unroll
        for (int dd = 0; dd < PASS; ++dd) {
#pragma unroll
          for (int i = 0; i < 4; ++i)
            if (okv[i]) sb[dd * G * SSTR + sto[i]] = acc[rw][dd][i];
        }
      }
      group_sync();
#pragma unroll
      for (int rw = 0; rw < 2; ++rw) {
        const float* sb = stg_g + rw * (SROWS * SSTR);
        const int y = yA + rw;
        if (y < H) {
          float* orow = obase + (size_t)rw * W + (size_t)(d0 * G) * plane;
#pragma unroll
          for (int k = 0; k < (SROWS * 8 + 127) / 128; ++k) {
            const int idx = tig + 128 * k;
            const int rowi = idx >> 3, quad = idx & 7;
            const int xq = cur.x0 + 4 * quad;
            if (rowi < nrow && xq < W) {
              float4 v = *reinterpret_cast<const float4*>(sb + rowi * SSTR + 4 * quad);
              if (slope <= 1.f) {
                v.x = fmaxf(v.x, v.x * slope); v.y = fmaxf(v.y, v.y * slope);
                v.z = fmaxf(v.z, v.z * slope); v.w = fmaxf(v.w, v.w * slope);
              } else {
                v.x = fminf(v.x, v.x * slope); v.y = fminf(v.y, v.y * slope);
                v.z = fminf(v.z, v.z * slope); v.w = fminf(v.w, v.w * slope);
              }
              float* op = orow + (size_t)rowi * plane + 4 * quad;
              if (ovec) {
                *reinterpret_cast<float4*>(op) = v;
              } else {
                op[0] = v.x;
                if (xq + 1 < W) op[1] = v.y;
                if (xq + 2 < W) op[2] = v.z;
                if (xq + 3 < W) op[3] = v.w;
              }
            }
          }
        }
      }
      group_sync();   // staging buffers are free again
    }

    // ---- 3. split / transpose the prefetched rows (a fresh strip is fetched here, after everybody left the ring) ----
    if (has_next) store_next(nxt, (s + 1) & 1, pe1, pe2, peh);
    cur = nxt;
    __syncthreads();
  }
}

// =====================================================================================================
// Host dispatch
// =====================================================================================================
static int launch_generic(const float* d1, const float* d2, float* out, int N, int C, int H, int W, int pad,
                          int ks, int md, int s1, int s2, int mul, int D, int OH, int OW, long long obs,
                          float slope, cudaStream_t st) {
  const long long total = (long long)N * D * OH * OW;
  const int threads = 256;
  long long blocks = (total + threads - 1) / threads;
  if (blocks > (long long)kNumSMs * 64) blocks = (long long)kNumSMs * 64;
  corr_generic_kernel<<<(unsigned)blocks, threads, 0, st>>>(d1, d2, out, N, C, H, W, pad, ks, md, s1, s2, mul,
                                                           D, OH, OW, obs, slope);
  return check_launch("corr_generic_kernel");
}

template <int MD>
static int launch_simt(const float* d1, const float* d2, float* out, int N, int C, int H, int W, long long obs,
                       float slope, cudaStream_t st) {
  using namespace simt;
  constexpr int G = 2 * MD + 1;
  const int tilesX = (W + TW - 1) / TW, tilesY = (H + TH - 1) / TH;
  const long long tiles = (long long)N * tilesX * tilesY;
  const size_t smem = sizeof(float) * CK * (TH * TW + (TH + 2 * MD) * (TW + 8));
  static SmemOptIn opt;
  {
    const cudaError_t e = ensure_dyn_smem(corr_simt_kernel<MD>, (int)smem, opt);
    if (e != cudaSuccess) return fail((int)e, "cudaFuncSetAttribute(corr_simt_kernel): %s", cudaGetErrorString(e));
  }
  corr_simt_kernel<MD><<<(unsigned)tiles, 64 * G, smem, st>>>(d1, d2, out, N, C, H, W, obs, slope);
  return check_launch(MD == 4 ? "corr_simt_kernel<4>" : "corr_simt_kernel<2>");
}

template <int MD, bool VEC>
static int launch_mma_impl(const float* d1, const float* d2, float* out, int N, int C, int H, int W,
                           long long obs, float slope, cudaStream_t st) {
  using namespace tc;
  const int tilesX = (W + TW - 1) / TW, tilesY = (H + TH - 1) / TH;
  const long long tiles = (long long)N * tilesX * tilesY;
  const int smem = smem_bytes(MD);
  static SmemOptIn opt;   // per template instantiation, per device
  {
    const cudaError_t e = ensure_dyn_smem(corr_mma_kernel<MD, VEC>, smem, opt);
    if (e != cudaSuccess) return fail((int)e, "cudaFuncSetAttribute(corr_mma_kernel): %s", cudaGetErrorString(e));
  }
  const int cap = tuning().corr_grid_cap > 0 ? tuning().corr_grid_cap : kNumSMs;
  const int grid = (int)(tiles < cap ? tiles : cap);
  corr_mma_kernel<MD, VEC><<<grid, NTHREADS, smem, st>>>(d1, d2, out, N, C, H, W, obs, slope, tilesX, tilesY,
                                                         (int)tiles);
  return check_launch(MD == 4 ? (VEC ? "corr_mma_kernel<4,vec>" : "corr_mma_kernel<4,scalar>")
                              : (VEC ? "corr_mma_kernel<2,vec>" : "corr_mma_kernel<2,scalar>"));
}

template <int MD, bool VEC>
static int launch_mma_ring_impl(const float* d1, const float* d2, float* out, int N, int C, int H, int W,
                                long long obs, float slope, cudaStream_t st) {
  using namespace r4;
  const int tilesX = (W + TW - 1) / TW, tilesY = (H + TH - 1) / TH;
  const long long tiles = (long long)N * tilesX * tilesY;
  const int smem = r4::smem_bytes(MD);
  const int ovec = ((W % 4) == 0 && (obs % 4) == 0 && aligned(out, 16)) ? 1 : 0;
  static SmemOptIn opt;
  {
    const cudaError_t e = ensure_dyn_smem(corr_mma_ring_kernel<MD, VEC>, smem, opt);
    if (e != cudaSuccess) return fail((int)e, "cudaFuncSetAttribute(corr_mma_ring_kernel): %s", cudaGetErrorString(e));
  }
  // strip-aligned work pieces: T = tiles per CTA if all SMs were used; each (n, x-strip) column is cut into
  // ceil(tilesY / T) pieces, one CTA per piece (e.g. level 2 of configs[1]: 64 strips x 2 pieces of 7 tiles = 128 CTAs)
  const int cap = tuning().corr_grid_cap > 0 ? tuning().corr_grid_cap : kNumSMs;
  const long long strips = (long long)N * tilesX;
  const int T = (int)((tiles + cap - 1) / cap);
  int pps = (tilesY + T - 1) / T;
  if (pps < 1) pps = 1;
  if (pps > tilesY) pps = tilesY;
  const unsigned grid = (unsigned)(strips * pps);
  corr_mma_ring_kernel<MD, VEC><<<grid, NTHREADS, smem, st>>>(d1, d2, out, N, C, H, W, obs, slope, tilesX, tilesY, pps,
                                                              ovec);
  // the reported names keep their ",th8" suffix so that logs and tests matching them do not change
  return check_launch(MD == 4 ? (VEC ? "corr_mma_ring_kernel<4,vec,th8>" : "corr_mma_ring_kernel<4,scalar,th8>")
                              : (VEC ? "corr_mma_ring_kernel<2,vec,th8>" : "corr_mma_ring_kernel<2,scalar,th8>"));
}

template <int MD>
static int launch_mma(const float* d1, const float* d2, float* out, int N, int C, int H, int W, long long obs,
                      float slope, cudaStream_t st) {
  const bool vec = (W % 4 == 0) && aligned(d2, 16) && aligned(d1, 16);
  if (tuning().corr_rb > 1) {   // tests: force the row-block kernel for every shape it can take
    const int rc = launch_corr_rb(MD, d1, d2, out, N, C, H, W, obs, slope, st);
    if (rc != -1) return rc;
  }
  if (C <= 32 && tuning().corr_tma) {   // TMA-in / TMA-out pipeline (corr_tma.cu); -1 = shape or alignment does not fit
    const int rc = launch_corr_tma(MD, d1, d2, out, N, C, H, W, obs, slope, st);
    if (rc != -1) return rc;
  }
  // row-block kernel (corr_rb.cu, all channels resident, one CTA per output row block): wins only on the smallest level
  // (level 6: 7 x 16, where the chunked tile kernel below has 16 tiles of 7 channel chunks); it was measured slower
  // elsewhere, so levels 3-5 stay on the tile kernel.
  if (tuning().corr_rb && C > 32 && (long long)N * H * W <= 1024) {
    const int rc = launch_corr_rb(MD, d1, d2, out, N, C, H, W, obs, slope, st);
    if (rc != -1) return rc;
  }
  if (C <= 32)   // strip-marching ring kernel: C <= 32 shapes the TMA kernel declines
    return vec ? launch_mma_ring_impl<MD, true>(d1, d2, out, N, C, H, W, obs, slope, st)
               : launch_mma_ring_impl<MD, false>(d1, d2, out, N, C, H, W, obs, slope, st);
  return vec ? launch_mma_impl<MD, true>(d1, d2, out, N, C, H, W, obs, slope, st)
             : launch_mma_impl<MD, false>(d1, d2, out, N, C, H, W, obs, slope, st);
}

}  // namespace mfn

extern "C" int mfn_correlation_forward(const float* data1, const float* data2, float* out, int N, int C, int H,
                                       int W, int pad_size, int kernel_size, int max_displacement, int stride1,
                                       int stride2, int is_multiply, long long out_batch_stride,
                                       float leaky_slope, int algo, void* stream) {
  using namespace mfn;
  MFN_REQUIRE(data1 && data2 && out, MFN_ERR_INVALID_ARG, "mfn_correlation_forward: null pointer");
  MFN_REQUIRE(N > 0 && C > 0 && H > 0 && W > 0, MFN_ERR_INVALID_ARG,
              "mfn_correlation_forward: non-positive extent (N=%d C=%d H=%d W=%d)", N, C, H, W);
  MFN_REQUIRE(kernel_size >= 1 && (kernel_size & 1), MFN_ERR_INVALID_ARG,
              "mfn_correlation_forward: kernel_size must be odd (got %d)", kernel_size);
  MFN_REQUIRE(stride1 >= 1 && stride2 >= 1 && max_displacement >= 0 && pad_size >= 0, MFN_ERR_INVALID_ARG,
              "mfn_correlation_forward: bad stride/displacement/pad");
  MFN_REQUIRE(aligned(data1, 4) && aligned(data2, 4) && aligned(out, 4), MFN_ERR_ALIGNMENT,
              "mfn_correlation_forward: pointers must be 4-byte aligned");
  const int kr = (kernel_size - 1) / 2, border = max_displacement + kr;
  const int ph = H + 2 * pad_size, pw = W + 2 * pad_size;
  const int OH = (ph - 2 * border + stride1 - 1) / stride1, OW = (pw - 2 * border + stride1 - 1) / stride1;
  MFN_REQUIRE(ph - 2 * border >= 1 && pw - 2 * border >= 1, MFN_ERR_INVALID_ARG,
              "mfn_correlation_forward: empty output");
  const int r = max_displacement / stride2, G = 2 * r + 1, D = G * G;
  const long long obs = out_batch_stride ? out_batch_stride : (long long)D * OH * OW;
  MFN_REQUIRE(obs >= (long long)D * OH * OW, MFN_ERR_INVALID_ARG, "mfn_correlation_forward: out_batch_stride too small");
  MFN_REQUIRE((long long)N * C * H * W < (1LL << 40) && (long long)C * H * W < (1LL << 31), MFN_ERR_ALIGNMENT,
              "mfn_correlation_forward: extents overflow kernel indexing");
  cudaStream_t st = as_stream(stream);
  const bool ref_regime = kernel_size == 1 && stride1 == 1 && stride2 == 1 && is_multiply &&
                          pad_size == max_displacement && (max_displacement == 4 || max_displacement == 2);
  if (algo == MFN_CORR_AUTO) algo = ref_regime ? (C >= 16 ? MFN_CORR_MMA_BF16X3 : MFN_CORR_SIMT) : MFN_CORR_GENERIC;
  switch (algo) {
    case MFN_CORR_GENERIC:
      return launch_generic(data1, data2, out, N, C, H, W, pad_size, kernel_size, max_displacement, stride1, stride2,
                            is_multiply ? 1 : 0, D, OH, OW, obs, leaky_slope, st);
    case MFN_CORR_SIMT:
      MFN_REQUIRE(ref_regime, MFN_ERR_UNSUPPORTED,
                  "mfn_correlation_forward: SIMT kernel needs kernel_size=1, strides=1, multiply, pad==md in {2,4}");
      return max_displacement == 4 ? launch_simt<4>(data1, data2, out, N, C, H, W, obs, leaky_slope, st)
                                   : launch_simt<2>(data1, data2, out, N, C, H, W, obs, leaky_slope, st);
    case MFN_CORR_MMA_BF16X3:
      MFN_REQUIRE(ref_regime, MFN_ERR_UNSUPPORTED,
                  "mfn_correlation_forward: MMA kernel needs kernel_size=1, strides=1, multiply, pad==md in {2,4}");
      return max_displacement == 4 ? launch_mma<4>(data1, data2, out, N, C, H, W, obs, leaky_slope, st)
                                   : launch_mma<2>(data1, data2, out, N, C, H, W, obs, leaky_slope, st);
    default:
      return fail(MFN_ERR_INVALID_ARG, "mfn_correlation_forward: unknown algo %d", algo);
  }
}
