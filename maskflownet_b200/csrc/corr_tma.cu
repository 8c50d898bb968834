// corr_tma.cu -- correlation cost-volume forward (K1), the production kernel for C <= 32 (level 2 of the S head and of the
// cascade: 55 % of the path's bytes).  sm_90a only.
//
// Serves mfn_correlation_forward (include/maskflow_b200.h) for the reference regime
//   F.Correlation(pad_size=md, kernel_size=1, max_displacement=md, stride1=1, stride2=1, is_multiply=1) + LeakyReLU
//   network/MaskFlownet.py:193-195,217 (md=4) and :440-441,467 (md=2).
//
// Design (one persistent CTA per SM, 15 warps, every stage decoupled from the next by mbarriers):
//
//   HBM --TMA tensor loads--> raw fp32 ring --converter warps--> split-bf16 rings --MMA warps--> staging --TMA tensor stores--> HBM
//
//   * work unit   = 4 image rows x 32 pixels of one (n, x-strip) column; a CTA owns a contiguous run of units in
//                   (strip, row-group) order (all SMs get the same number of units +-1) and marches down the strips.
//   * producer    (1 thread): cp.async.bulk.tensor 4-D loads of [8 channels][4 rows][40 px] data2 boxes (4-pixel x halo) and
//                   [8 channels][4 rows][32 px] data1 boxes straight from the NCHW tensors.  Out-of-image rows / columns /
//                   channels are zero-filled by the TMA unit: that IS the operator's pad_size, no padded temporaries.
//   * converters  (4 warps): fp32 -> (bf16 hi | bf16 lo), transposed to pixel-major 64 B / pixel rows with XOR-swizzled
//                   16-byte chunks (conflict-free STS.128 and ldmatrix, no padding); data1 pre-scaled by 1/C.  data2 rows
//                   live in a ring of 5 four-row quanta: every data2 row is fetched from HBM and converted exactly once
//                   per strip run (only the 25 % x halo is re-read, from L2).
//   * MMA warps   (2 groups x 4 warps; group = one unit, warp = 8-pixel block x 4 rows): banded formulation on
//                   mma.sync.m16n8k16 -- 16 data2 positions (M) x 8 pixels (N) x 16 channels (K) yields all 9 dx of those
//                   8 pixels for one dy; product = hi*lo + lo*hi + hi*hi, fp32 accumulate.  Because C <= 32 is ONE K chunk,
//                   an accumulator (row r, dy) is finished after its 6 MMAs: the warp walks the 12 data2 rows once, every
//                   ldmatrix'ed row feeds up to 4 pixel rows, accumulators live for 6 instructions (0.89 shared-memory
//                   wavefronts per MMA instead of 1.78 in the round-1 kernel).
//   * epilogue    LeakyReLU in registers, then 4 predicated STS.32 per accumulator tile into a [row][plane][32 px] staging
//                   slot laid out exactly as the 128B-swizzled TMA box (bank-conflict-free by construction: lanes j<2 store
//                   their even column first, lanes j>=2 their odd one); one cp.async.bulk.tensor store per (unit, dy)
//                   writes 9 planes x 4 rows x 128 B.  Image edges are clipped by the TMA unit.
#include <cuda.h>
#include <cuda_bf16.h>

#include "common.cuh"
#include "mma_tiles.cuh"
#include "ptx.cuh"

namespace mfn {
namespace ct {
constexpr int TW = 32, HX = 4, HWP = TW + 2 * HX, UR = 4, PXB = 64;
constexpr int F2_ROW = HWP * PXB;                 // 2560 bytes: one split row (hi or lo) of data2
constexpr int F1_ROW = TW * PXB;                  // 2048
constexpr int NQ = 5;                             // data2 ring: four-row quanta
constexpr int RING_LO = NQ * UR * F2_ROW, RING_BYTES = 2 * RING_LO;
constexpr int F1_LO = UR * F1_ROW, F1_STAGE = 2 * F1_LO;   // one data1 stage per MMA group
constexpr int RAW_F2 = 8 * UR * HWP * 4, RAW_F1 = 8 * UR * TW * 4, RAW_STAGE = RAW_F2 + RAW_F1, RAW_STAGES = 4;
constexpr int STG_SLOT = 5120, STG_SLOTS = 5;     // [4 rows][G planes][128 B] <= 4608, padded to the 1024-byte swizzle atom
constexpr int STG_BAR_FULL = 4608, STG_BAR_FREE = 4616;   // the slot's two mbarriers sit in its padding
constexpr int OFF_STG = 0, OFF_RING = OFF_STG + 2 * STG_SLOTS * STG_SLOT, OFF_F1 = OFF_RING + RING_BYTES,
              OFF_RAW = OFF_F1 + 2 * F1_STAGE, OFF_BAR = OFF_RAW + RAW_STAGES * RAW_STAGE;
constexpr int SMEM_BYTES = OFF_BAR + 512 + 1024;  // + barriers + slack for the manual 1024-byte alignment
constexpr int NCVT = 4, NMMA = 8;
constexpr int W_PROD = NCVT + NMMA, W_STORE = W_PROD + 1;
constexpr int NTHREADS = 32 * (NCVT + NMMA + 3);
enum {
  B_RAW_FULL = 0,
  B_RAW_EMPTY = B_RAW_FULL + RAW_STAGES,
  B_F2_FULL = B_RAW_EMPTY + RAW_STAGES,
  B_F2_EMPTY = B_F2_FULL + NQ,
  B_F1_FULL = B_F2_EMPTY + NQ,
  B_F1_EMPTY = B_F1_FULL + 2,
  B_COUNT = B_F1_EMPTY + 2
};
static_assert(B_COUNT * 8 <= 512, "barrier area");
static_assert(SMEM_BYTES <= 227 * 1024, "shared memory budget");

__device__ __forceinline__ void put_chunk(unsigned char* dst, int lo_off, const float (&e)[8], float sc) {
  uint4 hi, lo;
  split_pair(e[0] * sc, e[1] * sc, hi.x, lo.x);
  split_pair(e[2] * sc, e[3] * sc, hi.y, lo.y);
  split_pair(e[4] * sc, e[5] * sc, hi.z, lo.z);
  split_pair(e[6] * sc, e[7] * sc, hi.w, lo.w);
  *reinterpret_cast<uint4*>(dst) = hi;
  *reinterpret_cast<uint4*>(dst + lo_off) = lo;
}
}  // namespace ct

template <int MD>
__global__ void __launch_bounds__(ct::NTHREADS, 1)
    corr_tma_kernel(const __grid_constant__ CUtensorMap tm1, const __grid_constant__ CUtensorMap tm2,
                    const __grid_constant__ CUtensorMap tmo, int C, int Gs, int tilesX, int totalUnits, float slope) {
  using namespace ct;
  constexpr int G = 2 * MD + 1;
  constexpr int LR0 = 4 - MD;          // first local data2 row (of the 12 rows of quanta g-1, g, g+1) a unit touches
  constexpr int NLR = UR + 2 * MD;     // data2 rows a unit touches
  static_assert(UR * G * 128 <= STG_SLOT, "staging slot");

  extern __shared__ unsigned char smem_dyn[];
  const uint32_t dyn_u32 = smem_u32(smem_dyn);
  const uint32_t base = (dyn_u32 + 1023u) & ~1023u;
  unsigned char* sm = smem_dyn + (base - dyn_u32);
  const uint32_t bar0 = base + OFF_BAR;
  auto bar = [&](int idx) { return bar0 + 8u * (uint32_t)idx; };

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    for (int s = 0; s < RAW_STAGES; ++s) {
      mbar_init(bar(B_RAW_FULL + s), 1);
      mbar_init(bar(B_RAW_EMPTY + s), NCVT);
    }
    for (int s = 0; s < NQ; ++s) {
      mbar_init(bar(B_F2_FULL + s), NCVT);
      mbar_init(bar(B_F2_EMPTY + s), 12);   // 3 units x 4 warps (missing users at run ends are pre-arrived by the converter)
    }
    for (int s = 0; s < 2; ++s) {
      mbar_init(bar(B_F1_FULL + s), NCVT);
      mbar_init(bar(B_F1_EMPTY + s), 4);
    }
    for (int s = 0; s < 2 * STG_SLOTS; ++s) {
      mbar_init(base + OFF_STG + s * STG_SLOT + STG_BAR_FULL, 4);
      mbar_init(base + OFF_STG + s * STG_SLOT + STG_BAR_FREE, 1);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  // this CTA's run of units [U0, U0 + K) in (strip, row-group) order
  const int U0 = (int)(((long long)blockIdx.x * totalUnits) / gridDim.x);
  const int K = (int)(((long long)(blockIdx.x + 1) * totalUnits) / gridDim.x) - U0;
  if (K <= 0) return;
  const int s_first = U0 / Gs;

  if (warp == W_PROD) {
    // ============================== TMA PRODUCER ==============================
    if (lane == 0) {
      int i = 0;
      for (int k0 = 0; k0 < K;) {
        const int gu = U0 + k0, s = gu / Gs, g0 = gu - s * Gs;
        const int nm = min(K - k0, Gs - g0);
        const int n = s / tilesX, x0 = (s - n * tilesX) * TW;
        for (int j = 0; j < nm + 2; ++j, ++i) {
          const int y = UR * (g0 - 1 + j);
          const bool has_f1 = (j >= 1 && j <= nm);
#pragma unroll 1
          for (int cg = 0; cg < 4; ++cg) {
            const int seq = 4 * i + cg, rs = seq % RAW_STAGES, fill = seq / RAW_STAGES;
            mbar_wait(bar(B_RAW_EMPTY + rs), (fill & 1) ^ 1);
            const uint32_t dst = base + OFF_RAW + rs * RAW_STAGE;
            mbar_arrive_expect_tx(bar(B_RAW_FULL + rs), has_f1 ? RAW_STAGE : RAW_F2);
            tma_load_4d(dst, &tm2, x0 - HX, y, 8 * cg, n, bar(B_RAW_FULL + rs));
            if (has_f1) tma_load_4d(dst + RAW_F2, &tm1, x0, y, 8 * cg, n, bar(B_RAW_FULL + rs));
          }
        }
        k0 += nm;
      }
    }
  } else if (warp < NCVT) {
    // ============================== CONVERTERS ==============================
    const float invC = 1.f / (float)C;
    unsigned char* ring = sm + OFF_RING;
    const int hr = lane >> 3, hp = lane & 7, hpx = hp < HX ? hp : TW + hp;   // halo-column lane roles (4 rows x 8 px)
    int i = 0;
    for (int k0 = 0; k0 < K;) {
      const int gu = U0 + k0, s = gu / Gs, g0 = gu - s * Gs;
      const int nm = min(K - k0, Gs - g0);
      for (int j = 0; j < nm + 2; ++j, ++i) {
        const bool has_f1 = (j >= 1 && j <= nm);
        const int unit = k0 + j - 1;             // the unit whose data1 rows this quantum carries
        const int slot = i % NQ, qfill = i / NQ;
        mbar_wait(bar(B_F2_EMPTY + slot), (qfill & 1) ^ 1);
        if (warp == 0 && lane == 0) {
          const int nu = (j < nm ? 1 : 0) + ((j >= 1 && j - 1 < nm) ? 1 : 0) + ((j >= 2 && j - 2 < nm) ? 1 : 0);
          if (nu < 3) mbar_arrive_n(bar(B_F2_EMPTY + slot), 4u * (uint32_t)(3 - nu));
        }
        unsigned char* f1d = sm + OFF_F1 + (unit & 1) * F1_STAGE;
        if (has_f1) mbar_wait(bar(B_F1_EMPTY + (unit & 1)), ((unit >> 1) & 1) ^ 1);
#pragma unroll 1
        for (int cg = 0; cg < 4; ++cg) {
          const int seq = 4 * i + cg, rs = seq % RAW_STAGES, fill = seq / RAW_STAGES;
          mbar_wait(bar(B_RAW_FULL + rs), fill & 1);
          const float* r2 = reinterpret_cast<const float*>(sm + OFF_RAW + rs * RAW_STAGE);
          const float* r1 = r2 + RAW_F2 / 4;
          float e[8];
          // data2 row `warp`, pixels x0 .. x0+31 (raw index 4 + lane)
#pragma unroll
          for (int c = 0; c < 8; ++c) e[c] = r2[c * (UR * HWP) + warp * HWP + HX + lane];
          put_chunk(ring + (slot * UR + warp) * F2_ROW + swz(HX + lane, cg), RING_LO, e, 1.f);
          if (has_f1) {
#pragma unroll
            for (int c = 0; c < 8; ++c) e[c] = r1[c * (UR * TW) + warp * TW + lane];
            put_chunk(f1d + warp * F1_ROW + swz(lane, cg), F1_LO, e, invC);
          }
          if (warp == cg) {   // the two 4-pixel halo columns of all four rows
#pragma unroll
            for (int c = 0; c < 8; ++c) e[c] = r2[c * (UR * HWP) + hr * HWP + hpx];
            put_chunk(ring + (slot * UR + hr) * F2_ROW + swz(hpx, cg), RING_LO, e, 1.f);
          }
          __syncwarp();
          if (lane == 0) mbar_arrive(bar(B_RAW_EMPTY + rs));
        }
        if (lane == 0) {
          mbar_arrive(bar(B_F2_FULL + slot));
          if (has_f1) mbar_arrive(bar(B_F1_FULL + (unit & 1)));
        }
      }
      k0 += nm;
    }
  } else if (warp < NCVT + NMMA) {
    // ============================== MMA WARPS ==============================
    const int grp = (warp - NCVT) >> 2, b = (warp - NCVT) & 3;
    const int g = lane >> 2, j = lane & 3, e2 = j >> 1;
    const int l8 = lane & 7, mi = lane >> 3;
    const int sw = (l8 >> 1) & 3;
    uint32_t offA[2], offB[2];
#pragma unroll
    for (int kk = 0; kk < 2; ++kk) {
      offA[kk] = (uint32_t)((8 * b + 8 * (mi & 1) + l8) * PXB + (((2 * kk + (mi >> 1)) ^ sw) << 4));
      // data1 (B operand) rows are fetched in the pixel order 0 1 2 3 5 4 7 6: the accumulator columns (2j, 2j+1) of a lane
      // then ARE the pixels (2j + e2, 2j + 1 - e2) its two store slots take -- no register selects in the epilogue
      offB[kk] = (uint32_t)((8 * b + (l8 ^ ((l8 >> 2) & 1))) * PXB + (((2 * kk + (mi & 1)) ^ sw) << 4) + (mi >> 1) * F1_LO);
    }
    const uint32_t ring_u32 = base + OFF_RING, f1_u32 = base + OFF_F1 + grp * F1_STAGE;
    // Staging addresses.  Accumulator element (row, col) = f2 position 8b-4+row vs pixel 8b+col -> dx index row-col-4+MD.
    // Store slot S0 = element (g, 2j+e2), S1 = (g, 2j+1-e2), S2/S3 = the same columns of row g+8 (dx index + 8): within one
    // STS the lanes j<2 write even columns and the lanes j>=2 odd ones, which with the 128B swizzle hits 32 distinct banks.
    const int colS[2] = {2 * j + e2, 2 * j + 1 - e2};
    int pre[2][UR];
    bool ok[4];
#pragma unroll
    for (int q = 0; q < 2; ++q) {
      const int col = colS[q];
      const int dxi = g - col - 4 + MD;
      ok[q] = dxi >= 0 && dxi < G;
      ok[q + 2] = dxi + 8 >= 0 && dxi + 8 < G;
      const int chunk = 2 * b + (col >> 2);
#pragma unroll
      for (int r = 0; r < UR; ++r) {
        const int L = r * G + dxi;   // line of the slot ([row][plane] order); L + 8 has the same swizzle phase
        pre[q][r] = L * 128 + ((chunk ^ (L & 7)) << 4) + (col & 3) * 4;
      }
    }
    const uint32_t stg_u32 = base + OFF_STG + grp * (STG_SLOTS * STG_SLOT);
    unsigned char* stg = sm + OFF_STG + grp * (STG_SLOTS * STG_SLOT);

    // running staging-slot cursor: byte offset of the slot the NEXT new dy-group takes, and the parity of its fill
    int s_off = 0;
    uint32_t s_par = 0;
    for (int k = grp; k < K; k += 2) {
      const int gu = U0 + k, s = gu / Gs;
      const int a = k + 2 * (s - s_first);   // first quantum (stream index) of this unit
      // ---- B fragments (data1, pre-scaled): held in registers for the whole unit ----
      mbar_wait(bar(B_F1_FULL + grp), (k >> 1) & 1);
      uint32_t bq[UR][2][4];
#pragma unroll
      for (int r = 0; r < UR; ++r)
#pragma unroll
        for (int kk = 0; kk < 2; ++kk) ldsm_x4(f1_u32 + (uint32_t)(r * F1_ROW) + offB[kk], bq[r][kk]);
      __syncwarp();
      if (lane == 0) mbar_arrive(bar(B_F1_EMPTY + grp));
      uint32_t qrow[3], qbar[3];   // shared-memory address of the first row / the "empty" barrier of the unit's three quanta
#pragma unroll
      for (int t = 0; t < 3; ++t) {
        const int qi = a + t, qs = qi % NQ;
        mbar_wait(bar(B_F2_FULL + qs), (qi / NQ) & 1);
        qrow[t] = ring_u32 + (uint32_t)(qs * UR * F2_ROW);
        qbar[t] = bar(B_F2_EMPTY + qs);
      }
      auto frag = [&](int lr, uint32_t (&fh)[2][4], uint32_t (&fl)[2][4]) {
        const int qq = lr >> 2;
        const uint32_t ra = (qq == 0 ? qrow[0] : (qq == 1 ? qrow[1] : qrow[2])) + (uint32_t)((lr & 3) * F2_ROW);
#pragma unroll
        for (int kk = 0; kk < 2; ++kk) {
          ldsm_x4(ra + offA[kk], fh[kk]);
          ldsm_x4(ra + offA[kk] + RING_LO, fl[kk]);
        }
      };
      uint32_t ah[2][2][4], al[2][2][4];
      int win[UR];   // win[r] = slot offset of dy-group t - r (sliding window; pure register renaming once unrolled)
#pragma unroll
      for (int r = 0; r < UR; ++r) win[r] = 0;
      // One step = data2 row t (image row y0 - MD + t), serving pixel rows r with dy index d = t - r.  The G - 3 steps in
      // which all four pixel rows are served run as a RUNTIME loop (unrolled by two for the fragment double buffer); only
      // the three ramp-up and three ramp-down steps are unrolled with their compile-time row sets.  The fully unrolled walk
      // (12 x ~105 instructions, 20 KB) plus the other roles' code overflowed the instruction cache: the warps stalled
      // on instruction fetch.
      auto step = [&](const int t, const bool all, const uint32_t (&fh)[2][4], const uint32_t (&fl)[2][4], uint32_t (&nh)[2][4],
                      uint32_t (&nl)[2][4]) {
        if (t + 1 < NLR) frag(LR0 + t + 1, nh, nl);
#pragma unroll
        for (int r = UR - 1; r > 0; --r) win[r] = win[r - 1];
        if (all || t < G) {   // dy-group t starts: take the next slot once the TMA store of its previous tenant has drained it
          win[0] = s_off;
          mbar_wait(stg_u32 + (uint32_t)s_off + STG_BAR_FREE, s_par ^ 1u);
          s_off += STG_SLOT;
          if (s_off == STG_SLOTS * STG_SLOT) {
            s_off = 0;
            s_par ^= 1u;
          }
        }
        float acc[UR][4];
#pragma unroll
        for (int r = 0; r < UR; ++r)
#pragma unroll
          for (int q = 0; q < 4; ++q) acc[r][q] = 0.f;
#pragma unroll
        for (int kk = 0; kk < 2; ++kk) {
#pragma unroll
          for (int r = 0; r < UR; ++r)
            if (all || (t - r >= 0 && t - r < G)) mma_bf16(acc[r], fh[kk], bq[r][kk][2], bq[r][kk][3]);
#pragma unroll
          for (int r = 0; r < UR; ++r)
            if (all || (t - r >= 0 && t - r < G)) mma_bf16(acc[r], fl[kk], bq[r][kk][0], bq[r][kk][1]);
#pragma unroll
          for (int r = 0; r < UR; ++r)
            if (all || (t - r >= 0 && t - r < G)) mma_bf16(acc[r], fh[kk], bq[r][kk][0], bq[r][kk][1]);
        }
#pragma unroll
        for (int r = 0; r < UR; ++r) {
          if (!(all || (t - r >= 0 && t - r < G))) continue;
          float v[4];
#pragma unroll
          for (int q = 0; q < 4; ++q) v[q] = fmaxf(acc[r][q], acc[r][q] * slope);   // LeakyReLU for 0 <= slope <= 1
          unsigned char* sl = stg + win[r];
          if (ok[0]) *reinterpret_cast<float*>(sl + pre[0][r]) = v[0];
          if (ok[1]) *reinterpret_cast<float*>(sl + pre[1][r]) = v[1];
          if (ok[2]) *reinterpret_cast<float*>(sl + pre[0][r] + 1024) = v[2];
          if (ok[3]) *reinterpret_cast<float*>(sl + pre[1][r] + 1024) = v[3];
        }
        if (all || t >= UR - 1) {   // dy-group t - 3 received its last row from this warp
          asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
          __syncwarp();
          if (lane == 0) mbar_arrive(stg_u32 + (uint32_t)win[UR - 1] + STG_BAR_FULL);
        }
      };
      static_assert(UR == 4 && (G - 3) % 2 == 0 && NLR == G + 3, "step schedule");
      frag(LR0, ah[0], al[0]);
      step(0, false, ah[0], al[0], ah[1], al[1]);
      step(1, false, ah[1], al[1], ah[0], al[0]);
      step(2, false, ah[0], al[0], ah[1], al[1]);
#pragma unroll 1
      for (int t = UR - 1; t < G; t += 2) {
        step(t, true, ah[1], al[1], ah[0], al[0]);
        step(t + 1, true, ah[0], al[0], ah[1], al[1]);
      }
      step(G, false, ah[1], al[1], ah[0], al[0]);
      step(G + 1, false, ah[0], al[0], ah[1], al[1]);
      step(G + 2, false, ah[1], al[1], ah[0], al[0]);
      // ---- this warp no longer reads the unit's three quanta ----
      __syncwarp();
      if (lane == 0) {
#pragma unroll
        for (int t = 0; t < 3; ++t) mbar_arrive(qbar[t]);
      }
    }
  } else {
    // ============================== TMA STORE ISSUERS (one per MMA group) ==============================
    const int grp = warp - W_STORE;
    if (lane == 0) {
      int es = 0;
      for (int k = grp; k < K; k += 2) {
        const int gu = U0 + k, s = gu / Gs, g0 = gu - s * Gs;
        const int n = s / tilesX, x0 = (s - n * tilesX) * TW;
#pragma unroll 1
        for (int d = 0; d < G; ++d, ++es) {
          const int slot = es % STG_SLOTS, fill = es / STG_SLOTS;
          const uint32_t sa = base + OFF_STG + (grp * STG_SLOTS + slot) * STG_SLOT;
          mbar_wait(sa + STG_BAR_FULL, fill & 1);
          tma_store_4d(&tmo, sa, x0, d * G, UR * g0, n);
          bulk_commit();
          bulk_wait_read();
          mbar_arrive(sa + STG_BAR_FREE);
        }
      }
      bulk_wait_all();
    }
  }
}

// =====================================================================================================
// Host side: tensor maps (cuTensorMapEncodeTiled through the runtime's driver entry point: no link against libcuda)
// =====================================================================================================
EncodeTiledFn encode_tiled_fn() {
  static EncodeTiledFn fn = [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess ||
        q != cudaDriverEntryPointSuccess)
      p = nullptr;
    return reinterpret_cast<EncodeTiledFn>(p);
  }();
  return fn;
}

static int make_map(CUtensorMap* m, const void* ptr, const cuuint64_t (&dim)[4], const cuuint64_t (&stride_bytes)[3],
                    const cuuint32_t (&box)[4], CUtensorMapSwizzle swz) {
  EncodeTiledFn fn = encode_tiled_fn();
  if (!fn) return fail(MFN_ERR_UNSUPPORTED, "cuTensorMapEncodeTiled is not available from this driver");
  const cuuint32_t es[4] = {1, 1, 1, 1};
  const CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, const_cast<void*>(ptr), dim, stride_bytes, box, es,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, swz, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(MFN_ERR_UNSUPPORTED, "cuTensorMapEncodeTiled failed (CUresult %d)", (int)r);
  return MFN_OK;
}

// Returns -1 when the shape / alignment does not fit the TMA kernel (caller falls back), else the launch status.
template <int MD>
static int launch_corr_tma_impl(const float* d1, const float* d2, float* out, int N, int C, int H, int W, long long obs,
                                float slope, cudaStream_t st) {
  using namespace ct;
  constexpr int G = 2 * MD + 1;
  if (!(slope >= 0.f && slope <= 1.f)) return -1;   // the epilogue uses max(v, slope*v)
  if (C > 32 || (W % 4) != 0 || (obs % 4) != 0 || !aligned(d1, 16) || !aligned(d2, 16) || !aligned(out, 16)) return -1;
  if (encode_tiled_fn() == nullptr) return -1;
  CUtensorMap tm1, tm2, tmo;
  const cuuint64_t din[4] = {(cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)C, (cuuint64_t)N};
  const cuuint64_t sin[3] = {(cuuint64_t)W * 4, (cuuint64_t)W * H * 4, (cuuint64_t)W * H * C * 4};
  const cuuint32_t b1[4] = {TW, UR, 8, 1}, b2[4] = {HWP, UR, 8, 1};
  int rc = make_map(&tm1, d1, din, sin, b1, CU_TENSOR_MAP_SWIZZLE_NONE);
  if (rc) return rc;
  rc = make_map(&tm2, d2, din, sin, b2, CU_TENSOR_MAP_SWIZZLE_NONE);
  if (rc) return rc;
  // output viewed as (x, plane, y, n): the staging slot is [row][plane][32 px], 128B-swizzled
  const cuuint64_t dout[4] = {(cuuint64_t)W, (cuuint64_t)(G * G), (cuuint64_t)H, (cuuint64_t)N};
  const cuuint64_t sout[3] = {(cuuint64_t)W * H * 4, (cuuint64_t)W * 4, (cuuint64_t)obs * 4};
  const cuuint32_t bo[4] = {TW, G, UR, 1};
  rc = make_map(&tmo, out, dout, sout, bo, CU_TENSOR_MAP_SWIZZLE_128B);
  if (rc) return rc;

  static SmemOptIn opt;
  {
    const cudaError_t e = ensure_dyn_smem(corr_tma_kernel<MD>, SMEM_BYTES, opt);
    if (e != cudaSuccess) return fail((int)e, "cudaFuncSetAttribute(corr_tma_kernel): %s", cudaGetErrorString(e));
  }
  const int tilesX = (W + TW - 1) / TW, Gs = (H + UR - 1) / UR;
  const long long units = (long long)N * tilesX * Gs;
  if (units >= (1LL << 30)) return -1;
  const int cap = tuning().corr_grid_cap > 0 ? tuning().corr_grid_cap : kNumSMs;
  const int grid = (int)(units < cap ? units : cap);
  corr_tma_kernel<MD><<<grid, NTHREADS, SMEM_BYTES, st>>>(tm1, tm2, tmo, C, Gs, tilesX, (int)units, slope);
  return check_launch(MD == 4 ? "corr_tma_kernel<4>" : "corr_tma_kernel<2>");
}

int launch_corr_tma(int md, const float* d1, const float* d2, float* out, int N, int C, int H, int W, long long obs,
                    float slope, cudaStream_t st) {
  return md == 4 ? launch_corr_tma_impl<4>(d1, d2, out, N, C, H, W, obs, slope, st)
                 : launch_corr_tma_impl<2>(d1, d2, out, N, C, H, W, obs, slope, st);
}

}  // namespace mfn
