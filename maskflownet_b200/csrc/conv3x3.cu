// conv3x3.cu -- decoder dense-block convolution (SURVEY.md section 8f, row N2) for sm_90a.
//
// Serves mfn_conv3x3_forward: the 3x3 / stride 1 / pad 1 convolutions of the reference's decoder and context network
//   x = concat(leaky(convL_i(x)), x)        network/MaskFlownet.py:219-223, 237-241, ... (conv block: :166-175)
// reading its input channels IN PLACE from the level's concat buffer and writing bias + LeakyReLU'ed output channels into
// the slot in front of them (no concat copies).  fp32-accurate on tensor cores: activations and weights are split into
// bf16 hi + lo, each product is hi*hi + hi*lo + lo*hi (3 x mma.sync.m16n8k16, fp32 accumulate) -- the same scheme as the
// correlation kernel (corr_fwd.cu); relative error ~2^-17 per product, far inside TF32's 2^-11.
//
// Implicit GEMM, M = pixels, N = output channels, K = 9 * Cin walked as (32-channel chunk) x (tap):
//   * CTA = 8 warps = WR x WC; a warp owns one image row segment of 32 pixels (2 m16 tiles) x NTN n8 tiles of output
//     channels; CTA pixel tile = WR rows x 32 pixels.
//   * per chunk the (WR+2) x 40 pixel halo tile of the input is converted once into split-bf16, pixel-major, 64 B per pixel,
//     XOR-swizzled shared memory (lane = pixel loads: one 128-byte line per LDG); the nine taps are nine shifted ldmatrix
//     views of that tile -- no im2col.
//   * weights are pre-packed once (mfn_conv3x3_pack_weights) into per-(chunk, tap) tiles in exactly the shared-memory
//     image (hi | lo, swizzled), so the kernel streams them with 16-byte cp.async through a 3-stage ring.
#include "mma_tiles.cuh"

namespace mfn {
// packed weight image: [chunk q][tap t][hi | lo][f (Cout padded to 8)][64 B swizzled]: tile = 2 * CoutP * 64 bytes
__global__ void conv3x3_pack_kernel(const float* __restrict__ w, unsigned char* __restrict__ packed, int Cin, int Cout,
                                    int CoutP, int nChunks) {
  using namespace c3;
  const long long total = (long long)nChunks * 9 * CoutP * 16;  // (q, tap, f, channel pair)
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int j = (int)(i & 15);
    const int f = (int)((i >> 4) % CoutP);
    const int tap = (int)((i / (16LL * CoutP)) % 9);
    const int q = (int)(i / (16LL * CoutP * 9));
    const int c = 32 * q + 2 * j;
    float a = 0.f, b = 0.f;
    if (f < Cout) {
      if (c < Cin) a = w[((size_t)f * Cin + c) * 9 + tap];
      if (c + 1 < Cin) b = w[((size_t)f * Cin + c + 1) * 9 + tap];
    }
    uint32_t hi, lo;
    split_pair(a, b, hi, lo);
    unsigned char* tile = packed + ((size_t)q * 9 + tap) * (2 * CoutP * PXB);
    const int off = swz(f, j >> 2) + (j & 3) * 4;
    *reinterpret_cast<uint32_t*>(tile + off) = hi;
    *reinterpret_cast<uint32_t*>(tile + CoutP * PXB + off) = lo;
  }
}

// WC warp columns x NTN n8-tiles per warp cover the (padded) output channels; WR = 8 / WC image rows per CTA.
// PT = false: dilation 1, one halo tile per channel chunk serves all nine taps.
// PT = true : any dilation: each tap converts its own shifted WR x 32 tile (dilated taps do not share a compact halo).
template <int WC, int NTN, bool PT>
__global__ void __launch_bounds__(c3::NTHREADS, 1)
    conv3x3_mma_kernel(const float* __restrict__ x, long long x_bs, const unsigned char* __restrict__ wpack,
                       const float* __restrict__ bias, float* __restrict__ out, long long out_bs, int Cin, int H, int W,
                       int Cout, int CoutP, int nChunks, float slope, int tilesX, int tilesY, int dil, int lin_prefix) {
  using namespace c3;
  constexpr int WR = 8 / WC;
  constexpr int TROWS = PT ? WR : WR + 2;          // rows of the input tile
  constexpr int HWP = PT ? TW : c3::HWP;           // pixels per tile row
  constexpr int IN_LO = TROWS * HWP * PXB;         // byte offset of the lo image inside an input stage
  constexpr int IN_STAGE = 2 * IN_LO;
  const int WT_LO = CoutP * PXB;                   // lo image offset inside a weight tile
  const int WT_BYTES = 2 * WT_LO;

  extern __shared__ __align__(128) unsigned char smem[];
  unsigned char* in_s = smem;                       // [2][IN_STAGE]
  unsigned char* wt_s = smem + 2 * IN_STAGE;        // [WSTAGES][WT_BYTES]

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int wr = warp / WC, wc = warp % WC;         // warp's image row inside the tile / output-channel column
  const int tile = blockIdx.x;
  const int tx = tile % tilesX, ty = (tile / tilesX) % tilesY, n = tile / (tilesX * tilesY);
  const int x0 = tx * TW, y0 = ty * WR;
  const size_t plane = (size_t)H * W;
  const float* xn = x + (size_t)n * x_bs;

  // ---- input tile conversion: units of 32 lanes x 8 channels (lane = pixel).  main units: (row, 8-channel chunk) over the
  //      32 aligned pixels; halo-column units: (4 rows, chunk) over the 4 + 4 pixels left / right of them ----
  constexpr int U_MAIN = TROWS * 4;
  constexpr int U_HALO = PT ? 0 : ((TROWS + 3) / 4) * 4;
  constexpr int U_TOT = U_MAIN + U_HALO;
  constexpr int UPW = (U_TOT + 7) / 8;
  auto unit_geom = [&](int u, int& row, int& chunk, int& pidx, int& xx, bool& act) {
    act = u < U_TOT;
    if (u < U_MAIN) {
      row = u >> 2;
      chunk = u & 3;
      pidx = PT ? lane : HX + lane;
      xx = x0 + lane;
    } else {
      const int k = u - U_MAIN;
      row = 4 * (k >> 2) + (lane >> 3);
      chunk = k & 3;
      const int px8 = lane & 7;
      pidx = px8 < 4 ? px8 : TW + px8;             // 0..3 | 36..39
      xx = px8 < 4 ? x0 - HX + px8 : x0 + TW + (px8 - 4);
      act = act && row < TROWS;
    }
  };
  // PT: `q` is the iteration index (chunk * 9 + tap) and the tile is shifted by the tap's dilated offset
  auto load_tile = [&](int q, float (&e)[UPW][8]) {
    int sy = -1, sx = 0;
    if (PT) {
      const int tap = q % 9;
      sy = (tap / 3 - 1) * dil;
      sx = (tap % 3 - 1) * dil;
      q /= 9;
    }
#pragma unroll
    for (int k = 0; k < UPW; ++k) {
      int row, chunk, pidx, xx;
      bool act;
      unit_geom(warp * UPW + k, row, chunk, pidx, xx, act);
      xx += sx;
      const int yy = y0 + sy + row;
      const bool ok = act && yy >= 0 && yy < H && xx >= 0 && xx < W;
      const int c0 = 32 * q + 8 * chunk;
      const float* p = xn + (size_t)c0 * plane + (size_t)yy * W + xx;
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        e[k][c] = (ok && c0 + c < Cin) ? __ldg(p) : 0.f;
        p += plane;
      }
    }
  };
  auto store_tile = [&](int stage, const float (&e)[UPW][8]) {
#pragma unroll
    for (int k = 0; k < UPW; ++k) {
      int row, chunk, pidx, xx;
      bool act;
      unit_geom(warp * UPW + k, row, chunk, pidx, xx, act);
      if (!act) continue;
      uint4 hi, lo;
      split_pair(e[k][0], e[k][1], hi.x, lo.x);
      split_pair(e[k][2], e[k][3], hi.y, lo.y);
      split_pair(e[k][4], e[k][5], hi.z, lo.z);
      split_pair(e[k][6], e[k][7], hi.w, lo.w);
      unsigned char* dst = in_s + stage * IN_STAGE + row * (HWP * PXB) + swz(pidx, chunk);
      *reinterpret_cast<uint4*>(dst) = hi;
      *reinterpret_cast<uint4*>(dst + IN_LO) = lo;
    }
  };
  auto load_weights = [&](int it, int stage) {   // it = q * 9 + tap: contiguous tile in the packed image
    const unsigned char* src = wpack + (size_t)it * WT_BYTES;
    const uint32_t dst = smem_u32(wt_s + stage * WT_BYTES);
    for (int o = tid * 16; o < WT_BYTES; o += NTHREADS * 16) cp_async16(dst + o, src + o);
  };

  // ---- consumer lane constants ----
  const int g = lane >> 2, j = lane & 3;
  const int l8 = lane & 7, mi = lane >> 3;
  const int swB = (l8 >> 1) & 3;
  // B fragments: x4 = (n-tile pair member mi>>1, k-half mi&1): weight rows f = 8*(nt + (mi>>1)) + l8
  uint32_t offB[2];
#pragma unroll
  for (int kk = 0; kk < 2; ++kk) offB[kk] = (uint32_t)((8 * (mi >> 1) + l8) * PXB + (((2 * kk + (mi & 1)) ^ swB) << 4));
  const int fbase = wc * NTN * 8;                   // first output channel of this warp

  float acc[2][NTN][4];
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int nt = 0; nt < NTN; ++nt)
#pragma unroll
      for (int i = 0; i < 4; ++i) acc[mt][nt][i] = 0.f;

  const int nIter = nChunks * 9;
  // ---- prologue: input chunk 0 (PT: tile of iteration 0), weight tiles 0 and 1 ----
  {
    float e[UPW][8];
    load_tile(0, e);
    store_tile(0, e);
  }
  load_weights(0, 0);
  cp_async_commit();
  if (nIter > 1) load_weights(1, 1);
  cp_async_commit();

  const uint32_t in_u32 = smem_u32(in_s), wt_u32 = smem_u32(wt_s);
  float pe[UPW][8];
  for (int it = 0; it < nIter; ++it) {
    const int q = it / 9, tap = it - 9 * q;
    const int ky = tap / 3, kx = tap - 3 * ky;
    cp_async_wait<1>();          // weight tile `it` has landed (this thread's part)
    __syncthreads();             // ... everybody's part; the input tile is complete; the stages of iteration it-1 are free
    if (it + 2 < nIter) load_weights(it + 2, (it + 2) % WSTAGES);
    cp_async_commit();
    if (PT) {
      if (it + 1 < nIter) load_tile(it + 1, pe);                       // next tap's tile: in flight during this tap's MMAs
    } else {
      if (tap == 0 && q + 1 < nChunks) load_tile(q + 1, pe);           // next input chunk: global -> registers
      if (tap == 8 && q + 1 < nChunks) store_tile((q + 1) & 1, pe);    // ... -> split bf16 (read after the next barrier)
    }

    const uint32_t wst = wt_u32 + (uint32_t)((it % WSTAGES) * WT_BYTES);
    const uint32_t ist = PT ? in_u32 + (uint32_t)((it & 1) * IN_STAGE + wr * (HWP * PXB))
                            : in_u32 + (uint32_t)((q & 1) * IN_STAGE + (wr + ky) * (HWP * PXB));
    const bool half_chunk = 32 * q + 16 >= Cin;   // the upper 16 channels of the last chunk are padding: skip their MMAs
#pragma unroll
    for (int kk = 0; kk < 2; ++kk) {
      if (kk == 1 && half_chunk) break;
      uint32_t ah[2][4], al[2][4];
#pragma unroll
      for (int mt = 0; mt < 2; ++mt) {
        // A rows: 16 pixels x0 + 16*mt + (kx - 1) + r  ->  tile pixel index HX - 1 + kx + 16*mt + r  (PT: 16*mt + r)
        const int p = (PT ? 0 : HX - 1 + kx) + 16 * mt + 8 * (mi & 1) + l8;
        const uint32_t a = ist + (uint32_t)(p * PXB + (((2 * kk + (mi >> 1)) ^ ((p >> 1) & 3)) << 4));
        ldsm_x4(a, ah[mt]);
        ldsm_x4(a + IN_LO, al[mt]);
      }
#pragma unroll
      for (int nt = 0; nt < NTN; nt += 2) {
        uint32_t bh[4], bl[4];
        const uint32_t b = wst + (uint32_t)((fbase + 8 * nt) * PXB) + offB[kk];
        ldsm_x4(b, bh);
        ldsm_x4(b + WT_LO, bl);
#pragma unroll
        for (int mt = 0; mt < 2; ++mt) {
          mma_bf16(acc[mt][nt], ah[mt], bl[0], bl[1]);
          mma_bf16(acc[mt][nt], al[mt], bh[0], bh[1]);
          mma_bf16(acc[mt][nt], ah[mt], bh[0], bh[1]);
          if (nt + 1 < NTN) {
            mma_bf16(acc[mt][nt + 1], ah[mt], bl[2], bl[3]);
            mma_bf16(acc[mt][nt + 1], al[mt], bh[2], bh[3]);
            mma_bf16(acc[mt][nt + 1], ah[mt], bh[2], bh[3]);
          }
        }
      }
    }
    if (PT && it + 1 < nIter) store_tile((it + 1) & 1, pe);   // stage (it+1)&1 was last read in iteration it-1
  }

  // ---- epilogue: bias + LeakyReLU, NCHW stores (8 consecutive pixels x 4 bytes = one sector per (plane, instruction)) ----
  const int y = y0 + wr;
  if (y >= H) return;
  float* on = out + (size_t)n * out_bs + (size_t)y * W;
#pragma unroll
  for (int nt = 0; nt < NTN; ++nt) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int f = fbase + 8 * nt + 2 * j + (i & 1);
      if (f >= Cout) continue;
      const float b = bias ? __ldg(bias + f) : 0.f;
#pragma unroll
      for (int mt = 0; mt < 2; ++mt) {
        const int xx = x0 + 16 * mt + g + 8 * (i >> 1);
        if (xx < W) on[(size_t)f * plane + xx] = leaky(acc[mt][nt][i] + b, f < lin_prefix ? 1.f : slope);
      }
    }
  }
}

template <int WC, int NTN, bool PT>
static int launch_conv_impl(const float* x, long long x_bs, const unsigned char* wpack, const float* bias, float* out,
                            long long out_bs, int N, int Cin, int H, int W, int Cout, int dil, float slope, int lin_prefix,
                            cudaStream_t st) {
  using namespace c3;
  constexpr int WR = 8 / WC;
  const int CoutP = cout_pad(Cout);
  const int nChunks = (Cin + 31) / 32;
  const int tilesX = (W + TW - 1) / TW, tilesY = (H + WR - 1) / WR;
  const int in_stage = PT ? 2 * WR * TW * PXB : 2 * (WR + 2) * HWP * PXB;
  const int smem = 2 * in_stage + WSTAGES * 2 * CoutP * PXB;
  static SmemOptIn opt;
  {
    const cudaError_t e = ensure_dyn_smem(conv3x3_mma_kernel<WC, NTN, PT>, smem, opt);
    if (e != cudaSuccess) return fail((int)e, "cudaFuncSetAttribute(conv3x3_mma_kernel): %s", cudaGetErrorString(e));
  }
  const unsigned grid = (unsigned)((long long)N * tilesX * tilesY);
  conv3x3_mma_kernel<WC, NTN, PT><<<grid, NTHREADS, smem, st>>>(x, x_bs, wpack, bias, out, out_bs, Cin, H, W, Cout,
                                                               CoutP, nChunks, slope, tilesX, tilesY, dil, lin_prefix);
  return check_launch(PT ? "conv3x3_mma_kernel<per-tap tiles>" : "conv3x3_mma_kernel<halo tile>");
}

template <int WC, int NTN>
static int launch_conv(const float* x, long long x_bs, const unsigned char* wpack, const float* bias, float* out,
                       long long out_bs, int N, int Cin, int H, int W, int Cout, int dil, float slope, int lin_prefix,
                       cudaStream_t st) {
  return dil == 1 ? launch_conv_impl<WC, NTN, false>(x, x_bs, wpack, bias, out, out_bs, N, Cin, H, W, Cout, 1, slope, lin_prefix, st)
                  : launch_conv_impl<WC, NTN, true>(x, x_bs, wpack, bias, out, out_bs, N, Cin, H, W, Cout, dil, slope, lin_prefix, st);
}

// bytes of the mma.sync weight image (first region of the packed buffer; the wgmma image follows it)
long long conv3x3_sync_packed_bytes(int Cin, int Cout) {
  if (Cout > 128) return 0;   // the mma.sync kernels stop at 128 output channels; wider layers exist only in the wgmma image
  return (long long)((Cin + 31) / 32) * 9 * 2 * c3::cout_pad(Cout) * c3::PXB;
}

}  // namespace mfn

extern "C" long long mfn_conv3x3_packed_bytes(int Cin, int Cout) {
  if (Cin <= 0 || Cout <= 0) return 0;
  return mfn::conv3x3_sync_packed_bytes(Cin, Cout) + mfn::conv3x3_wgmma_packed_bytes(Cin, Cout);
}

extern "C" int mfn_conv3x3_pack_weights(const float* weight, void* packed, int Cin, int Cout, void* stream) {
  using namespace mfn;
  MFN_REQUIRE(weight && packed, MFN_ERR_INVALID_ARG, "mfn_conv3x3_pack_weights: null pointer");
  MFN_REQUIRE(Cin > 0 && Cout > 0, MFN_ERR_INVALID_ARG, "mfn_conv3x3_pack_weights: non-positive extent");
  MFN_REQUIRE(aligned(packed, 16), MFN_ERR_ALIGNMENT, "mfn_conv3x3_pack_weights: packed buffer must be 16-byte aligned");
  MFN_REQUIRE(Cout <= 256, MFN_ERR_UNSUPPORTED, "mfn_conv3x3_pack_weights: at most 256 output channels (got %d)", Cout);
  if (Cout <= 128) {
    const int CoutP = c3::cout_pad(Cout), nChunks = (Cin + 31) / 32;
    const long long total = (long long)nChunks * 9 * CoutP * 16;
    long long blocks = (total + 255) / 256;
    if (blocks > 4096) blocks = 4096;
    conv3x3_pack_kernel<<<(unsigned)blocks, 256, 0, as_stream(stream)>>>(weight, static_cast<unsigned char*>(packed), Cin,
                                                                         Cout, CoutP, nChunks);
    const int rc = check_launch("conv3x3_pack_kernel");
    if (rc) return rc;
  }
  return conv3x3_wgmma_pack(weight, static_cast<unsigned char*>(packed) + conv3x3_sync_packed_bytes(Cin, Cout), Cin, Cout,
                           as_stream(stream));
}

extern "C" int mfn_conv3x3_forward(const float* x, long long x_batch_stride, const void* packed_weight,
                                   const float* bias, float* out, long long out_batch_stride, int N, int Cin, int H,
                                   int W, int Cout, int dilation, float leaky_slope, void* stream) {
  return mfn_conv3x3_forward_ex(x, x_batch_stride, packed_weight, bias, out, out_batch_stride, N, Cin, H, W, Cout, 1,
                                dilation, MFN_CONV_OUT_NCHW, leaky_slope, stream);
}

extern "C" int mfn_conv3x3_forward_ex(const float* x, long long x_batch_stride, const void* packed_weight,
                                      const float* bias, float* out, long long out_batch_stride, int N, int Cin, int H,
                                      int W, int Cout, int stride, int dilation, int out_mode, float leaky_slope,
                                      void* stream) {
  return mfn_conv3x3_forward_ws(x, x_batch_stride, packed_weight, bias, out, out_batch_stride, N, Cin, H, W, Cout, stride,
                                dilation, out_mode, leaky_slope, nullptr, 0, stream);
}

extern "C" long long mfn_conv3x3_workspace_bytes(int N, int Cin, int H, int W, int Cout, int stride, int dilation) {
  using namespace mfn;
  if (N <= 0 || Cin <= 0 || H <= 0 || W <= 0 || Cout <= 0 || Cout > 256 || dilation < 1 ||
      !(stride == 1 || (stride == 2 && dilation == 1)))
    return 0;
  if (!tuning().conv_wgmma && Cout <= 128 && stride == 1) return 0;   // mma.sync kernel
  return conv3x3_wgmma_workspace_bytes(N, Cin, H, W, Cout, stride, dilation);
}

extern "C" int mfn_conv3x3_forward_ws(const float* x, long long x_batch_stride, const void* packed_weight,
                                      const float* bias, float* out, long long out_batch_stride, int N, int Cin, int H,
                                      int W, int Cout, int stride, int dilation, int out_mode, float leaky_slope,
                                      void* workspace, long long workspace_bytes, void* stream) {
  using namespace mfn;
  MFN_REQUIRE(workspace_bytes >= 0 && (workspace || workspace_bytes == 0) && aligned(workspace, 16), MFN_ERR_INVALID_ARG,
              "mfn_conv3x3_forward_ws: workspace must be 16-byte aligned (or null with 0 bytes)");
  MFN_REQUIRE(x && packed_weight && out, MFN_ERR_INVALID_ARG, "mfn_conv3x3_forward: null pointer");
  MFN_REQUIRE(N > 0 && Cin > 0 && H > 0 && W > 0 && Cout > 0, MFN_ERR_INVALID_ARG,
              "mfn_conv3x3_forward: non-positive extent");
  MFN_REQUIRE(Cout <= 256, MFN_ERR_UNSUPPORTED, "mfn_conv3x3_forward: at most 256 output channels (got %d)", Cout);
  MFN_REQUIRE(dilation >= 1, MFN_ERR_INVALID_ARG, "mfn_conv3x3_forward: dilation must be >= 1");
  MFN_REQUIRE(stride == 1 || (stride == 2 && dilation == 1), MFN_ERR_UNSUPPORTED,
              "mfn_conv3x3_forward: stride must be 1, or 2 with dilation 1 (got stride %d, dilation %d)", stride, dilation);
  MFN_REQUIRE(aligned(packed_weight, 16), MFN_ERR_ALIGNMENT, "mfn_conv3x3_forward: packed weights must be 16-byte aligned");
  const int bf16 = out_mode & MFN_CONV_BF16;   // passed on to the wgmma kernel, the only one with the bf16 variant
  out_mode &= ~MFN_CONV_BF16;
  const int lin_prefix = out_mode >> 8, mode = out_mode & 0xff;
  MFN_REQUIRE(mode == MFN_CONV_OUT_NCHW || (mode == MFN_CONV_OUT_DEPTH_TO_SPACE2 && stride == 1 && Cout % 4 == 0),
              MFN_ERR_INVALID_ARG, "mfn_conv3x3_forward: depth-to-space output needs stride 1 and Cout %% 4 == 0");
  MFN_REQUIRE(lin_prefix >= 0 && lin_prefix <= Cout && (lin_prefix == 0 || mode == MFN_CONV_OUT_NCHW), MFN_ERR_INVALID_ARG,
              "mfn_conv3x3_forward: linear prefix (out_mode >> 8 = %d) needs NCHW output and <= Cout", lin_prefix);
  const int OH = (H - 1) / stride + 1, OW = (W - 1) / stride + 1;
  const long long xbs = x_batch_stride ? x_batch_stride : (long long)Cin * H * W;
  const long long obs = out_batch_stride ? out_batch_stride : (long long)Cout * OH * OW;
  MFN_REQUIRE(xbs >= (long long)Cin * H * W && obs >= (long long)Cout * OH * OW, MFN_ERR_INVALID_ARG,
              "mfn_conv3x3_forward: batch stride smaller than the tensor");
  const unsigned char* wp = static_cast<const unsigned char*>(packed_weight);
  cudaStream_t st = as_stream(stream);
  const bool sync_ok = Cout <= 128 && stride == 1 && mode == MFN_CONV_OUT_NCHW;   // what the mma.sync kernels cover
  if (tuning().conv_wgmma || !sync_ok) {   // wgmma kernel
    const int rc = conv3x3_wgmma_launch(x, xbs, wp + conv3x3_sync_packed_bytes(Cin, Cout), bias, out, obs, N, Cin, H, W,
                                       Cout, stride, dilation, out_mode | bf16, leaky_slope, st, 0,
                                       static_cast<float*>(workspace), workspace_bytes);
    if (rc != -1) return rc;
    MFN_REQUIRE(sync_ok, MFN_ERR_UNSUPPORTED, "mfn_conv3x3_forward: shape fits neither kernel (Cout=%d stride=%d dilation=%d)",
                Cout, stride, dilation);
  }
  MFN_REQUIRE(!bf16, MFN_ERR_UNSUPPORTED,
              "mfn_conv3x3_forward: MFN_CONV_BF16 runs on the wgmma kernel only, and this launch would take the mma.sync "
              "kernel (tuning conv_wgmma = 0, or a shape the wgmma kernel declines)");
  const int nt = (Cout + 7) / 8;   // n8 tiles needed
  if (nt <= 4) return launch_conv<1, 4>(x, xbs, wp, bias, out, obs, N, Cin, H, W, Cout, dilation, leaky_slope, lin_prefix, st);
  if (nt <= 8) return launch_conv<1, 8>(x, xbs, wp, bias, out, obs, N, Cin, H, W, Cout, dilation, leaky_slope, lin_prefix, st);
  if (nt <= 12) return launch_conv<2, 6>(x, xbs, wp, bias, out, obs, N, Cin, H, W, Cout, dilation, leaky_slope, lin_prefix, st);
  return launch_conv<2, 8>(x, xbs, wp, bias, out, obs, N, Cin, H, W, Cout, dilation, leaky_slope, lin_prefix, st);
}

extern "C" int mfn_conv3x3_forward_split(const void* x, int x_channels, int x_c0, const void* packed_weight,
                                         const float* bias, float* out, long long out_batch_stride, void* out_split,
                                         int out_split_channels, int out_split_c0, int N, int Cin, int H, int W, int Cout,
                                         int dilation, int out_mode, float leaky_slope, void* workspace,
                                         long long workspace_bytes, void* stream) {
  using namespace mfn;
  MFN_REQUIRE(workspace_bytes >= 0 && (workspace || workspace_bytes == 0) && aligned(workspace, 16), MFN_ERR_INVALID_ARG,
              "mfn_conv3x3_forward_split: workspace must be 16-byte aligned (or null with 0 bytes)");
  const int bf16 = out_mode & MFN_CONV_BF16;   // x and out_split are bf16 activations
  out_mode &= ~MFN_CONV_BF16;
  const int lin_prefix = out_mode >> 8, mode = out_mode & 0xff;
  MFN_REQUIRE(x && packed_weight && (out || (out_split && lin_prefix == 0)), MFN_ERR_INVALID_ARG,
              "mfn_conv3x3_forward_split: null pointer");
  MFN_REQUIRE(N > 0 && Cin > 0 && H > 0 && W > 0 && Cout > 0 && Cout <= 256 && dilation >= 1, MFN_ERR_INVALID_ARG,
              "mfn_conv3x3_forward_split: bad extent, Cout (<= 256) or dilation");
  // the last chunk loads whole 16-channel groups: past the slice they must be the buffer's zero pad, not its next channels
  MFN_REQUIRE(x_c0 >= 0 && x_c0 % 16 == 0 && x_c0 + Cin <= x_channels &&
                  ((x_c0 + Cin) % 16 == 0 || x_c0 + Cin == x_channels),
              MFN_ERR_INVALID_ARG,
              "mfn_conv3x3_forward_split: input slice [%d, %d) of the %d channels must start at a multiple of 16 and end "
              "at one or at the last channel", x_c0, x_c0 + Cin, x_channels);
  MFN_REQUIRE(aligned(packed_weight, 16) && aligned(x, 16), MFN_ERR_ALIGNMENT,
              "mfn_conv3x3_forward_split: packed weights and split input must be 16-byte aligned");
  MFN_REQUIRE(lin_prefix >= 0 && lin_prefix <= Cout && (lin_prefix == 0 || mode == MFN_CONV_OUT_NCHW), MFN_ERR_INVALID_ARG,
              "mfn_conv3x3_forward_split: linear prefix needs NCHW / split output and <= Cout");
  MFN_REQUIRE(mode == MFN_CONV_OUT_NCHW || (mode == MFN_CONV_OUT_DEPTH_TO_SPACE2 && Cout % 4 == 0 && !out_split),
              MFN_ERR_INVALID_ARG, "mfn_conv3x3_forward_split: depth-to-space output needs Cout %% 4 == 0 and fp32 output");
  const int Fo = out_split ? lin_prefix : (mode ? Cout / 4 : Cout), OS = mode ? 4 : 1;
  const long long obs = out_batch_stride ? out_batch_stride : (long long)Fo * H * W * OS;
  MFN_REQUIRE(obs >= (long long)Fo * H * W * OS, MFN_ERR_INVALID_ARG, "mfn_conv3x3_forward_split: batch stride too small");
  SplitIO sio;
  sio.in = x;
  sio.in_C = x_channels;
  sio.in_c0 = x_c0;
  sio.out = out_split;
  sio.out_C = out_split_channels;
  sio.out_c0 = out_split_c0;
  const unsigned char* wp = static_cast<const unsigned char*>(packed_weight);
  const int rc = conv3x3_wgmma_launch(nullptr, 0, wp + conv3x3_sync_packed_bytes(Cin, Cout), bias, out, obs, N, Cin, H, W,
                                      Cout, 1, dilation, out_mode | bf16, leaky_slope, as_stream(stream), 0,
                                      static_cast<float*>(workspace), workspace_bytes, sio);
  MFN_REQUIRE(rc != -1, MFN_ERR_UNSUPPORTED,
              "mfn_conv3x3_forward_split: unsupported (odd dilation >= 2, split output slice not 16-channel aligned "
              "after an even linear prefix, or too large)");
  return rc;
}
