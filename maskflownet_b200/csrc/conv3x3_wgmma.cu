// conv3x3_wgmma.cu -- the 3x3 convolutions of the decoder, the context network and the feature pyramid (SURVEY.md section
// 8f, row N2) on the Hopper tensor cores: warpgroup MMAs (wgmma.mma_async) with the accumulators in registers.  Contract as
// in conv3x3.cu (channel slices of a level buffer in, bias + LeakyReLU'ed channel slice out, fp32-accurate through the bf16
// hi/lo split: three MMAs hi*lo + lo*hi + hi*hi per product); reference call sites network/MaskFlownet.py:147-300.
//
// Implicit GEMM without im2col:   D[pixel, f] = sum_{tap, c} X[pixel + tap offset, c] * Wt[tap][c][f]
//   * a work tile is R = 2 image rows x MT consecutive output pixels x (up to 128) output channels; MT = 128, or 64 where
//     the output is at most 64 pixels wide (levels 4-6) and at stride 2 (tile_width).  PERSISTENT kernel, one CTA per SM, tiles dealt round-robin; the
//     producers / weight loader run ahead across tile boundaries.
//   * K is walked as (16-channel chunk) x (tap).  Per chunk the producer warps convert the input rows the nine taps touch
//     from fp32 NCHW into split bf16 in the *no-swizzle K-major core-matrix layout*: plane [8-channel group][pixel] with
//     16 bytes per entry.  In that layout a tap shift is nothing but a different start address (+16 bytes per pixel), so
//     all nine taps are nine shared-memory descriptors over ONE converted tile: (start, LBO = plane pitch, SBO = 128 B).
//     Stride 2 de-interleaves even / odd pixels so the same holds (see the geometry helpers).  Where a tensor map fits
//     the fp32 input (stride 1 on 128-pixel tiles, stride 2 on 64-pixel ones, dilation 1), one thread first stages the
//     raw rows in shared memory with TMA and the producers convert from there (SplitDev::in == 2, raw_pitch).
//   * weights are pre-packed (mfn_conv3x3_pack_weights) into per-(chunk, tap) images of the same layout and streamed by
//     one thread with 1-D bulk copies (cp.async.bulk + mbarrier complete_tx) through a deep ring (up to 24 stages).
//   * two consumer warpgroups, one per output row, each issue m64nNk16 MMAs (bf16 x bf16 -> fp32) for the MT / 64
//     64-pixel blocks of their row; after each tap's group they wait for the previous group and release the weight / input
//     stages it read, and at the end of a tile apply bias + LeakyReLU and store NCHW -- through shared-memory staging
//     rows and asynchronous bulk copies when the output rows are 16-byte aligned, else from registers -- or, for the
//     transposed convolutions, scatter 2x2 sub-pixel phases (depth-to-space).
//   * layers wider than 128 output channels are cut into two 128-channel work items per tile (register budget).
//   * TERMS (template argument) = products per multiply-add: 3 is the hi/lo split above; 1 is the opt-in bf16 mode
//     (MFN_CONV_BF16): only A_hi x B_hi, the input stage holds the hi plane alone, the weight ring streams the hi half of
//     the same packed image, and split outputs are bf16 activations (one plane, split_act.cuh).
#include <cstring>
#include <type_traits>

#include "mma_tiles.cuh"
#include "split_act.cuh"

namespace mfn {
namespace um {
// pixels per tile row MT (template argument of the kernel): 128 = two 64-row wgmma M blocks per output row; outputs at most
// 64 pixels wide (levels 4-6) take MT = 64, one M block per row, so that no MMA is issued for pixels right of the image.
// Stride 2 takes MT = 64 too while the TMA-staged input is on: its raw ring only fits beside 64-pixel tiles (smem_map).
constexpr int MT_WIDE = 128, MT_NARROW = 64;
inline int tile_width(int OW, int stride) {
  return tuning().conv_narrow && (OW <= MT_NARROW || (stride == 2 && tuning().conv_tma_in)) ? MT_NARROW : MT_WIDE;
}
constexpr int R = 2;             // output rows per CTA tile
constexpr int NTHREADS = 384;    // warps 0..3: row-0 warpgroup, 4..7: row-1 warpgroup, 8: weight loader, 9..11: producers
constexpr int NCONS = 8;         // consumer warps: each arrives once on every stage it releases
constexpr int NPROD = 3;         // producer warps
constexpr int MAX_AS = 4, MAX_WS = 24;
constexpr int MAX_RS = 4;        // raw fp32 input stages of the TMA-staged input path (SplitDev::in == 2)
constexpr int BATCH = 6;         // producer items (32 entries x 8 channels) in flight per warp
constexpr int BAR_BYTES = 1024;  // a_full/a_empty [MAX_AS], w_full/w_empty [MAX_WS], r_full/r_empty [MAX_RS]

// Geometry of the converted input tile: `nslots` image rows of PW entries each.
//   stride 1 (any dilation d): rows y0 - d .. y0 + R - 1 + d (or the 3R rows the taps touch when d >= R); entry p of a row is
//     pixel x0 - d + p; tap (ky, kx) of output row r starts at entry slot(r, ky) * PW + kx * d.
//   stride 2 (d = 1): rows 2 y0 - 1 .. 2 y0 + 2R - 1; a row is de-interleaved into its even pixels 2 (x0 + p), p < MT, and
//     its odd pixels 2 (x0 - 1 + p - MT) + 1, p >= MT, so that "next output pixel" is again "next entry": tap kx reads
//     the odd block from 0 (kx = 0), the even block (kx = 1) or the odd block from 1 (kx = 2).
__host__ __device__ inline int n_slots(int stride, int dil) { return stride == 2 ? 2 * R + 1 : (dil >= R ? 3 * R : R + 2 * dil); }
__host__ __device__ inline int row_pitch(int mt, int stride, int dil) { return stride == 2 ? 2 * mt + 1 : mt + 2 * dil; }
__host__ __device__ inline int slot_of(int r, int ky, int stride, int dil) {
  return stride == 2 ? 2 * r + ky : (dil >= R ? ky * R + r : r + ky * dil);
}
__host__ __device__ inline int tap_xoff(int mt, int kx, int stride, int dil) {
  return stride == 2 ? (kx == 1 ? 0 : (kx == 0 ? mt : mt + 1)) : kx * dil;
}
// ext = 2 ("band" mode of K3 through linearity, warp_lin.cu): the input is a VIRTUAL image of (n + 6) rows / columns --
// the n real ones followed by [0, 0, first, 0, 0, last] -- so that ONE convolution also yields the 1-D convolutions of the
// first / last row and column and the four corner pixels that the MXNet-1.5 border rule needs.  Maps a virtual
// coordinate to the real one, or -1 (zero).
__host__ __device__ inline int band_map(int v, int n) { return v < n ? v : (v == n + 2 ? 0 : (v == n + 5 ? n - 1 : -1)); }
// TMA-staged fp32 input (dilation 1, no ext): one raw stage is a tensor box of fp32, [channel][row][pixel], that starts
// and ends on 16-byte boundaries of the image row (x0, the tile's first output pixel, is a multiple of MT):
//   stride 1: {MT + 8 pixels from x0 - 4, the nslots rows, 16 channels}; entry p of converted row s (pixel x0 - 1 + p)
//     reads raw[c][s][p + 3].
//   stride 2 (MT = 64): {2 MT + 4 pixels from 2 x0 - 4, the 5 rows, 8 channels}, one 8-channel plane of the chunk per
//     stage; even entry p < MT (pixel 2 (x0 + p)) reads raw[c][s][2 p + 4], odd entry p >= MT (pixel
//     2 (x0 - 1 + p - MT) + 1) reads raw[c][s][2 (p - MT) + 3].
__host__ __device__ inline int raw_pitch(int mt, int stride) { return stride == 2 ? 2 * mt + 4 : mt + 8; }
__host__ __device__ inline int raw_channels(int stride) { return stride == 2 ? 8 : 16; }
__host__ __device__ inline int raw_stage_bytes(int nslots, int mt, int stride) {
  return raw_channels(stride) * nslots * raw_pitch(mt, stride) * 4;
}
// most raw stages the ring may take: stride 1 keeps the 2 it was measured with; stride 2, whose 8-channel stages hold less
// (conv1a's 3 channels: 8 KB of image per stage), deepens the ring while >= 3 weight stages still fit (smem_map)
__host__ __device__ inline int raw_ring_max(int stride) { return stride == 2 ? MAX_RS : 2; }
// output channels padded to the next multiple of 16 up to 128 (the MMA widths this file instantiates); wider layers to
// 256 = 2 x 128
__host__ __device__ inline int cout_pad(int cout) { return cout <= 128 ? (cout + 15) / 16 * 16 : 256; }
// Narrow layers (N <= 64) fold the hi / lo weight images into ONE operand of 2N rows:
//   D[:, 0:2N] += A_hi x [B_hi ; B_lo]      (N' = 2N)        D[:, 0:N] += A_lo x B_hi
// two MMAs per product instead of three, and one A read fewer from shared memory; the epilogue adds the two column blocks.
__host__ __device__ inline bool fold_hi_lo(int CoutP) { return CoutP <= 64; }
// Taps per weight-ring stage (compile-time variants of the kernel).  Both rings are bound by their ROUND-TRIP latency
// (release -> mbarrier -> waiting thread wakes -> copy / conversion -> mbarrier -> consumer wakes), not by bandwidth: a ring
// of S stages delivers S stages per round trip.  Narrow layers, whose MMAs per tap are short, therefore move 9 / 3 taps
// per bulk copy.
__host__ __device__ inline int taps_per_stage(int CoutP) { return CoutP <= 32 ? 9 : (CoutP <= 64 ? 3 : 1); }

// wgmma shared-memory descriptor, no swizzle (layout type 0), K-major: 8-row x 16-byte core matrices; SBO = distance
// between 8-row groups (M/N direction), LBO = distance between the two 8-element K groups of one k16 MMA.
__device__ __forceinline__ uint64_t desc_hi(uint32_t lbo_bytes, uint32_t sbo_bytes) {
  return ((uint64_t)((lbo_bytes >> 4) & 0x3FFFu) << 16) | ((uint64_t)((sbo_bytes >> 4) & 0x3FFFu) << 32);
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator reads / writes across the asynchronous MMAs
template <int S>
__device__ __forceinline__ void fence_acc(float (&d)[S]) {
#pragma unroll
  for (int i = 0; i < S; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// m64nNk16, A and B from shared memory (K-major), D += A B (scale_d = 0: D = A B); uses d[0 .. N/2 - 1]
template <int S>
__device__ __forceinline__ void wgmma_n16(float (&d)[S], uint64_t a, uint64_t b, uint32_t scale_d) {
  static_assert(S >= 8, "accumulator too small");
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
      : "l"(a), "l"(b), "r"(scale_d));
}
template <int S>
__device__ __forceinline__ void wgmma_n32(float (&d)[S], uint64_t a, uint64_t b, uint32_t scale_d) {
  static_assert(S >= 16, "accumulator too small");
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(a), "l"(b), "r"(scale_d));
}
template <int S>
__device__ __forceinline__ void wgmma_n48(float (&d)[S], uint64_t a, uint64_t b, uint32_t scale_d) {
  static_assert(S >= 24, "accumulator too small");
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %26, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n48k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23}, %24, %25, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23])
      : "l"(a), "l"(b), "r"(scale_d));
}
template <int S>
__device__ __forceinline__ void wgmma_n64(float (&d)[S], uint64_t a, uint64_t b, uint32_t scale_d) {
  static_assert(S >= 32, "accumulator too small");
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(a), "l"(b), "r"(scale_d));
}
template <int S>
__device__ __forceinline__ void wgmma_n80(float (&d)[S], uint64_t a, uint64_t b, uint32_t scale_d) {
  static_assert(S >= 40, "accumulator too small");
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %42, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n80k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39}, %40, %41, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39])
      : "l"(a), "l"(b), "r"(scale_d));
}
template <int S>
__device__ __forceinline__ void wgmma_n96(float (&d)[S], uint64_t a, uint64_t b, uint32_t scale_d) {
  static_assert(S >= 48, "accumulator too small");
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %50, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n96k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47}, %48, %49, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47])
      : "l"(a), "l"(b), "r"(scale_d));
}
template <int S>
__device__ __forceinline__ void wgmma_n112(float (&d)[S], uint64_t a, uint64_t b, uint32_t scale_d) {
  static_assert(S >= 56, "accumulator too small");
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %58, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n112k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55}, %56, %57, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55])
      : "l"(a), "l"(b), "r"(scale_d));
}
template <int S>
__device__ __forceinline__ void wgmma_n128(float (&d)[S], uint64_t a, uint64_t b, uint32_t scale_d) {
  static_assert(S >= 64, "accumulator too small");
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(a), "l"(b), "r"(scale_d));
}
template <int N, int S>
__device__ __forceinline__ void wgmma_bf16(float (&d)[S], uint64_t a, uint64_t b, uint32_t scale_d) {
  if constexpr (N == 16) wgmma_n16(d, a, b, scale_d);
  else if constexpr (N == 32) wgmma_n32(d, a, b, scale_d);
  else if constexpr (N == 48) wgmma_n48(d, a, b, scale_d);
  else if constexpr (N == 64) wgmma_n64(d, a, b, scale_d);
  else if constexpr (N == 80) wgmma_n80(d, a, b, scale_d);
  else if constexpr (N == 96) wgmma_n96(d, a, b, scale_d);
  else if constexpr (N == 112) wgmma_n112(d, a, b, scale_d);
  else wgmma_n128(d, a, b, scale_d);
}

// Split-K plan (host: plan_split): work items [0, from) are whole tiles, the tiles [from, numTiles) are cut into k parts
// over the channel chunks.  Their raw sums go to ws[part][n - n_lo][Cout][y - y_lo (rh rows)][OW].  ns = 2: every such
// item is further cut into two 128-channel halves (consecutive work indices).
struct SplitK {
  int k, from, n_lo, y_lo, rh;
  long long part_stride;
  float* ws;
  // tile -> (n, ty, tx) without integer division: ceil(2^32 / (tilesX tilesY)) and ceil(2^32 / tilesX), or 0 when the
  // products could overflow the exactness bound (then the kernel divides)
  uint32_t magic_tp, magic_tx;
  int as_wide;   // input stages of the wide (single-tap weight stage) layers: 3 or 2 (smem_map)
  int ns;        // output-channel halves per tile: 1, or 2 for CoutP = 256
  int stg;       // bytes of the staged epilogue's shared-memory rows; 0: whole tiles store from registers
};
__device__ __forceinline__ void decode_tile(int tile, int tilesX, int tilesY, const SplitK& sk, int& tx, int& ty, int& n) {
  if (sk.magic_tp) {
    n = (int)__umulhi((uint32_t)tile, sk.magic_tp);
    const int rem = tile - n * tilesX * tilesY;
    ty = sk.magic_tx ? (int)__umulhi((uint32_t)rem, sk.magic_tx) : rem;   // magic_tx == 0: tilesX == 1
    tx = rem - ty * tilesX;
  } else {
    tx = tile % tilesX;
    ty = (tile / tilesX) % tilesY;
    n = tile / (tilesX * tilesY);
  }
}
// split-activation operands on the device (SplitIO): in = 1: the input tiles are copied row by row from in_buf (groups
// in_g0.. of a buffer of in_Cg groups per plane); in = 2: fp32 input whose raw tiles the tensor map {W, H, Cin, N} stages
// in shared memory for the producers to convert; in = 0: fp32 input the producers load themselves.  out != null = output channels
// >= the linear prefix go to channel out_c0.. of a split buffer of out_Cg groups
struct SplitDev {
  int in, in_g0, in_Cg;
  const unsigned char* in_buf;
  unsigned char* out;
  int out_Cg, out_c0;
};
struct Work {
  int tile, part, cb, ce, nh;   // part < 0: a whole tile; nh: output-channel half
};
__device__ __forceinline__ Work decode_work(int w, const SplitK& sk, int nChunks) {
  Work r;
  r.nh = 0;
  if (sk.ns == 2) {
    r.nh = w & 1;
    w >>= 1;
  }
  if (sk.k <= 1 || w < sk.from) {
    r.tile = w; r.part = -1; r.cb = 0; r.ce = nChunks;
  } else {
    const int u = w - sk.from, t = u / sk.k;
    r.tile = sk.from + t;
    r.part = u - t * sk.k;
    r.cb = r.part * nChunks / sk.k;
    r.ce = (r.part + 1) * nChunks / sk.k;
  }
  return r;
}

struct SmemMap {
  int a_lo, a_stage, w_tile, w_stage, w_off, bar_off, stg_off, total, AS, WS, raw_off, raw_stage, RS;
};
// staged epilogue: per consumer warpgroup STG_CH output channels x MT pixels of fp32, row pitch SPITCH floats (the 4-float
// pad makes the fragment stores bank-conflict-free and keeps every row 16-byte aligned for the bulk copies; the 64-pixel
// tiles use the first half of each row)
constexpr int STG_CH = 32, SPITCH = MT_WIDE + 4;
constexpr int STG_BYTES = R * STG_CH * SPITCH * 4;
// stage counts from the shared-memory budget: 3 input stages when that still leaves >= 8 weight stages, else 2.
// stg: bytes of the epilogue staging rows (0 = the layer stores from registers).  terms = 1: the input and weight stages
// hold the hi images alone (half the bytes; w_tile is then the hi tile [2 planes][CoutP][16 B] in shared memory, while
// the packed image in global memory keeps its 64 CoutP bytes per tap).  raw: bytes of one raw fp32 input stage of the
// TMA-staged input path (0: none); its RS raw stages (the most up to rs_max that leave >= 3 weight stages, at least 2)
// follow the input stages at a 128-byte boundary (tensor-copy destinations), and the producers, whose conversion from
// shared memory is short, keep 2 input stages.
__host__ __device__ inline SmemMap smem_map(int E, int CoutP, int as_wide = 3, int stg = 0, int terms = 3, int raw = 0,
                                            int rs_max = 2) {
  SmemMap m;
  m.a_lo = 2 * E * 16;              // hi image: two 8-channel planes of E entries
  m.a_stage = terms == 1 ? m.a_lo : 2 * m.a_lo;   // hi (+ lo)
  m.w_tile = terms == 1 ? 32 * CoutP : 64 * CoutP;   // [hi (| lo)][2 planes][CoutP][16 B]
  int budget = 227 * 1024 - BAR_BYTES - stg;
  m.w_stage = taps_per_stage(CoutP) * m.w_tile;
  m.RS = 0;
  if (raw) {
    const int raw_off = (2 * m.a_stage + 127) / 128 * 128;
    m.RS = rs_max;
    while (m.RS > 2 && budget - raw_off - m.RS * raw < 3 * m.w_stage) --m.RS;
    budget -= m.RS * raw + (raw_off - 2 * m.a_stage);
  }
  // input stages: narrow layers (several taps per weight stage) take 4 when >= 4 weight stages still fit; wide layers keep
  // the weight ring deep (their weight stages are single taps) and take 3
  if (raw)
    m.AS = 2;
  else if (taps_per_stage(CoutP) > 1)
    m.AS = (4 * m.a_stage + 4 * m.w_stage <= budget) ? 4 : ((3 * m.a_stage + 3 * m.w_stage <= budget) ? 3 : 2);
  else   // as_wide = 2 would trade an input stage for four more single-tap weight stages; the launcher passes 3
    m.AS = (as_wide >= 3 && 3 * m.a_stage + 8 * m.w_stage <= budget) ? 3 : 2;
  int ws = (budget - m.AS * m.a_stage) / m.w_stage;
  m.WS = ws > MAX_WS ? MAX_WS : ws;
  m.raw_off = raw ? (m.AS * m.a_stage + 127) / 128 * 128 : m.AS * m.a_stage;
  m.raw_stage = raw;
  m.w_off = m.raw_off + m.RS * raw;
  m.bar_off = m.w_off + m.WS * m.w_stage;
  m.stg_off = m.bar_off + BAR_BYTES;
  m.total = m.stg_off + stg;
  return m;
}
}  // namespace um

// wgmma weight image: [16-channel chunk c][tap][hi | lo][8-channel plane kc][f (CoutP)][8 x bf16 = 16 bytes]
// (narrow layers: [chunk][tap][plane][hi f.. | lo f..][16 bytes], see fold_hi_lo)
__global__ void conv3x3_pack_wgmma_kernel(const float* __restrict__ w, unsigned char* __restrict__ packed, int Cin, int Cout,
                                          int CoutP, int nChunks16) {
  const long long total = (long long)nChunks16 * 9 * CoutP * 8;   // (c, tap, f, channel pair)
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int j = (int)(i & 7);                     // channel pair inside the chunk
    const int f = (int)((i >> 3) % CoutP);
    const int tap = (int)((i / (8LL * CoutP)) % 9);
    const int c = (int)(i / (8LL * CoutP * 9));
    const int ch = 16 * c + 2 * j;
    float a = 0.f, b = 0.f;
    if (f < Cout) {
      if (ch < Cin) a = w[((size_t)f * Cin + ch) * 9 + tap];
      if (ch + 1 < Cin) b = w[((size_t)f * Cin + ch + 1) * 9 + tap];
    }
    uint32_t hi, lo;
    split_pair(a, b, hi, lo);
    const int wt = 64 * CoutP;
    unsigned char* tile = packed + ((size_t)c * 9 + tap) * wt;
    if (um::fold_hi_lo(CoutP)) {   // [8-channel plane][hi rows | lo rows][16 B]
      const int off = (j >> 2) * (2 * CoutP * 16) + f * 16 + (j & 3) * 4;
      *reinterpret_cast<uint32_t*>(tile + off) = hi;
      *reinterpret_cast<uint32_t*>(tile + CoutP * 16 + off) = lo;
    } else {                       // [hi | lo][8-channel plane][rows][16 B]
      const int off = (j >> 2) * (CoutP * 16) + f * 16 + (j & 3) * 4;
      *reinterpret_cast<uint32_t*>(tile + off) = hi;
      *reinterpret_cast<uint32_t*>(tile + wt / 2 + off) = lo;
    }
  }
}

// NW: accumulator columns per 64-pixel block (FOLD and TERMS = 3: 2 x CoutP, else CoutP or 128 per channel half).
// FOLD: the packed image has the folded layout (CoutP <= 64).  TERMS: 3 (hi/lo split) or 1 (bf16: hi x hi only).
// MT: pixels per tile row, 128 or 64 (um::tile_width).
template <int NW, bool FOLD, int TPS, int TERMS, int MT>
__global__ void __launch_bounds__(um::NTHREADS, 1)
    conv3x3_wgmma_kernel(const float* __restrict__ x, long long x_bs, const unsigned char* __restrict__ wpack,
                         const float* __restrict__ bias_arg, float* __restrict__ out_base, long long out_bs, int Cin, int H, int W,
                         int OH, int OW, int Cout, int CoutP, int nChunks, float slope_arg, int tilesX, int tilesY, int numWork,
                         int stride, int dil, int out_mode_arg, int ext, um::SplitK sk, um::SplitDev xs,
                         const __grid_constant__ CUtensorMap tmx, int dbg) {
  using namespace um;
  // out_mode_arg = mode | (linear_prefix << 8): the first linear_prefix output channels are written WITHOUT the activation
  // (a second, linear head sharing the input pass of an activated layer: network.py folds pred_flow / pred_mask over the
  // dense block's input into its last convolution)
  // Split-K (sk.k > 1): `numWork` counts WORK ITEMS.  Items below sk.from are whole tiles; the tiles from sk.from on are
  // cut into sk.k parts over the channel chunks -- part p walks chunks [p nChunks / k, (p + 1) nChunks / k) and writes its
  // RAW partial sums (no bias, no activation) to the workspace; conv3x3_wgmma_reduce_kernel finishes that region.
  // dbg (tuning "conv_dbg", profiling only, results invalid): 2 = producers skip their global loads, 4 = no epilogue
  // stores, 8 = no MMAs, 16 = producers skip loads, conversion and shared-memory stores (they only hand over each stage),
  // 32 = the weight loader issues no bulk copies (it only hands over each weight stage); the barrier protocol is
  // unchanged, so each phase can be timed by removing it.
  static_assert(TERMS == 1 || TERMS == 3, "one or three products per multiply-add");
  static_assert(MT == MT_WIDE || MT == MT_NARROW, "128- or 64-pixel tile rows");
  constexpr bool FOLD_ACC = FOLD && TERMS == 3;   // the accumulator holds the [hi*hi | hi*lo] column blocks
  constexpr int P = TERMS == 1 ? 1 : 2;           // planes of the input stage and of a split output
  constexpr int NCOL = FOLD_ACC ? NW / 2 : NW;    // output channels per work item
  constexpr int MB = MT / 64;                     // m64 blocks per output row
  const int out_mode_k = out_mode_arg & 0xff, lin_prefix_k = out_mode_arg >> 8;
  extern __shared__ __align__(128) unsigned char smem[];
  const int nslots = n_slots(stride, dil), PW = row_pitch(MT, stride, dil), E = nslots * PW;
  const SmemMap sm = smem_map(E, CoutP, sk.as_wide, sk.stg, TERMS, xs.in == 2 ? raw_stage_bytes(nslots, MT, stride) : 0,
                              raw_ring_max(stride));
  const int AS = sm.AS, WS = sm.WS, RS = sm.RS;
  const uint32_t s_base = smem_u32(smem);
  const uint32_t bar0 = s_base + sm.bar_off;
  const uint32_t a_full = bar0, a_empty = bar0 + 8 * MAX_AS, w_full = bar0 + 16 * MAX_AS, w_empty = w_full + 8 * MAX_WS;
  const uint32_t r_full = w_empty + 8 * MAX_WS, r_empty = r_full + 8 * MAX_RS;

  const int tid = threadIdx.x, lane = tid & 31;
  const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0);   // warp-uniform role (keeps the wgmma path non-divergent)
  const size_t plane = (size_t)H * W;

  if (tid == 0) {
    for (int i = 0; i < AS; ++i) {
      mbar_init(a_full + 8 * i, xs.in == 1 ? 1 : NPROD);
      mbar_init(a_empty + 8 * i, NCONS);
    }
    for (int i = 0; i < RS; ++i) {
      mbar_init(r_full + 8 * i, 1);
      mbar_init(r_empty + 8 * i, NPROD);
    }
    for (int i = 0; i < WS; ++i) {
      mbar_init(w_full + 8 * i, 1);
      mbar_init(w_empty + 8 * i, NCONS);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp < 8) {
    // ============================ consumers: warpgroup r computes output row r of the tile ============================
    const int r = warp >> 2, wq = warp & 3;
    const uint32_t a_lbo = (uint32_t)E * 16u, b_lbo = (uint32_t)(FOLD_ACC ? 2 * CoutP : CoutP) * 16u;
    // descriptor low words (address >> 4) of the nine taps live in registers (the tap loop is fully unrolled)
    uint32_t a_off[9];
#pragma unroll
    for (int tap = 0; tap < 9; ++tap)
      a_off[tap] = (uint32_t)(slot_of(r, tap / 3, stride, dil) * PW + tap_xoff(MT, tap % 3, stride, dil));
    const uint64_t dh_a = desc_hi(a_lbo, 128u), dh_b = desc_hi(b_lbo, 128u);
    uint32_t as = 0, aph = 0, ws = 0, wph = 0;
    const uint32_t a_lo16 = (uint32_t)sm.a_lo >> 4, a_stage16 = (uint32_t)sm.a_stage >> 4, s_base16 = s_base >> 4;
    const uint32_t w_base16 = (s_base + (uint32_t)sm.w_off) >> 4, w_tile16 = (uint32_t)sm.w_tile >> 4, w_half16 = w_tile16 >> 1;
    const uint32_t w_stage16 = (uint32_t)sm.w_stage >> 4;
    // stages read by the previous MMA group, released once that group has completed (-1: none)
    int rel_w = -1, rel_a = -1;
    auto release = [&]() {
      if (lane == 0) {
        if (rel_w >= 0) mbar_arrive(w_empty + 8 * rel_w);
        if (rel_a >= 0) mbar_arrive(a_empty + 8 * rel_a);
      }
      rel_w = rel_a = -1;
    };
    float acc[MB][NW / 2];
    for (int work = blockIdx.x; work < numWork; work += gridDim.x) {
      const Work wk = decode_work(work, sk, nChunks);
      const int cb = wk.cb, ce = wk.ce;
      const uint32_t b_nh16 = (uint32_t)(wk.nh * NCOL);   // first weight row of this channel half (16 B rows)
#pragma unroll
      for (int mh = 0; mh < MB; ++mh) fence_acc(acc[mh]);
      if (dbg & 8) {   // profiling: the same barrier traffic without MMAs
        for (int c = cb; c < ce; ++c) {
          mbar_wait(a_full + 8 * as, aph);
          for (int tap = 0; tap < 9; ++tap) {
            if (tap % TPS == 0) mbar_wait(w_full + 8 * ws, wph);
            release();
            if (tap % TPS == TPS - 1) {
              rel_w = (int)ws;
              if (++ws == (uint32_t)WS) { ws = 0; wph ^= 1; }
            }
            if (tap == 8) rel_a = (int)as;
          }
          if (++as == (uint32_t)AS) { as = 0; aph ^= 1; }
        }
      }
      for (int c = (dbg & 8) ? ce : cb; c < ce; ++c) {
        mbar_wait(a_full + 8 * as, aph);
        const uint32_t a_st16 = s_base16 + as * a_stage16;
#pragma unroll
        for (int tap = 0; tap < 9; ++tap) {
          if (tap % TPS == 0) mbar_wait(w_full + 8 * ws, wph);
          const uint32_t w16 = w_base16 + ws * w_stage16 + (uint32_t)(tap % TPS) * w_tile16 + b_nh16;
          const uint64_t b_hi = dh_b | (uint64_t)w16, b_lo = dh_b | (uint64_t)(w16 + w_half16);
          const uint32_t sc = (tap == 0 && c == cb) ? 0u : 1u;
          wgmma_fence();
#pragma unroll
          for (int mh = 0; mh < MB; ++mh) {
            const uint32_t a16 = a_st16 + a_off[tap] + (uint32_t)(64 * mh);
            const uint64_t a_hi = dh_a | (uint64_t)a16, a_lo = dh_a | (uint64_t)(a16 + a_lo16);
            if constexpr (TERMS == 1) {
              wgmma_bf16<NW>(acc[mh], a_hi, b_hi, sc);
            } else if constexpr (FOLD) {
              wgmma_bf16<NW>(acc[mh], a_hi, b_hi, sc);       // [hi*hi | hi*lo]
              wgmma_bf16<NW / 2>(acc[mh], a_lo, b_hi, 1u);   // += lo*hi into the first block
            } else {
              wgmma_bf16<NW>(acc[mh], a_hi, b_lo, sc);
              wgmma_bf16<NW>(acc[mh], a_lo, b_hi, 1u);
              wgmma_bf16<NW>(acc[mh], a_hi, b_hi, 1u);
            }
          }
          wgmma_commit();
          wgmma_wait<1>();   // the previous tap's group has read its operands
          release();
          if (tap % TPS == TPS - 1) {
            rel_w = (int)ws;
            if (++ws == (uint32_t)WS) { ws = 0; wph ^= 1; }
          }
          if (tap == 8) rel_a = (int)as;
        }
        if (++as == (uint32_t)AS) { as = 0; aph ^= 1; }
      }
      wgmma_wait<0>();
#pragma unroll
      for (int mh = 0; mh < MB; ++mh) fence_acc(acc[mh]);
      release();

      // ---- epilogue from registers: m64nN accumulator fragment of thread (warp wq, lane): rows 16 wq + lane / 4 (+ 8),
      // columns 8 j + 2 (lane % 4) (+ 1) in registers 4 j + {0, 1} (+ {2, 3} for the row + 8)
      int tx, ty, n;
      decode_tile(wk.tile, tilesX, tilesY, sk, tx, ty, n);
      // a part of a split tile: raw sums into its slot of the workspace region [n_lo.., all channels, y_lo.., OW]
      const bool partial = wk.part >= 0;
      const float* const bias = partial ? nullptr : bias_arg;
      const float slope = partial ? 1.f : slope_arg;
      const int out_mode = partial ? 0 : out_mode_k, lin_prefix = partial ? 0 : lin_prefix_k;
      const size_t oplane0 = partial ? (size_t)sk.rh * OW : (size_t)OH * OW;    // plane pitch of plain NCHW output
      float* const out = partial ? sk.ws + (size_t)wk.part * (size_t)sk.part_stride + (size_t)(n - sk.n_lo) * Cout * oplane0 -
                                       (size_t)sk.y_lo * OW
                                 : out_base + (size_t)n * out_bs;
      const int y = ty * R + r;
      const int F = Cout >> 2;
      const size_t oplane2 = (size_t)(2 * OH) * (2 * OW);
      if (y < OH && !(dbg & 4) && sk.stg && !partial) {
        // staged epilogue (plain NCHW output, 16-byte aligned rows): SCH channels at a time, the warpgroup writes
        // bias + LeakyReLU'ed values into its staging rows ([channel][pixel], pitch SPITCH: conflict-free), and one thread
        // per channel hands the row segment to a bulk copy (full 128-byte lines, asynchronous: the global writes drain
        // while the next work item's MMAs run).  A piece waits only until the copies of the previous one have READ it.
        constexpr int SCH = NCOL % STG_CH == 0 ? STG_CH : 16;   // channels per piece (divides NCOL: a multiple of 16)
        float* const stg = reinterpret_cast<float*>(smem + sm.stg_off) + r * STG_CH * SPITCH;
        const int t = wq * 32 + lane;   // thread of this warpgroup
        const int x0 = tx * MT;
        const uint32_t seg = (uint32_t)((OW - x0 < MT ? OW - x0 : MT) * 4);
        if (xs.out != nullptr) {
          // split output (no linear prefix): the piece's SCH / 8 groups x P planes ({hi, lo}, or hi alone) are staged as
          // rows of MT 16-byte entries -- exactly their layout in global memory, one contiguous row segment each -- and
          // leave by one bulk copy per row.  A warp's pair stores cover 8 pixels x 4 words: 32 distinct banks.
          unsigned char* const sst = reinterpret_cast<unsigned char*>(stg);
#pragma unroll
          for (int pc = 0; pc < NCOL / SCH; ++pc) {
            if (t < SCH * P / 8) bulk_wait_read();
            named_bar_sync(1 + r, 128);
#pragma unroll
            for (int jj = 0; jj < SCH / 8; ++jj) {
              const int j = pc * (SCH / 8) + jj;
              const int f = wk.nh * NCOL + 8 * j + 2 * (lane & 3);
              const float b0 = (bias != nullptr && f < Cout) ? __ldg(bias + f) : 0.f;
              const float b1 = (bias != nullptr && f + 1 < Cout) ? __ldg(bias + f + 1) : 0.f;
              unsigned char* const row = sst + (P * jj * MT + 16 * wq + (lane >> 2)) * 16 + (lane & 3) * 4;
#pragma unroll
              for (int mh = 0; mh < MB; ++mh)
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                  const int i = 4 * j + 2 * h;
                  float v0 = acc[mh][i], v1 = acc[mh][i + 1];
                  if constexpr (FOLD_ACC) {
                    v0 += acc[mh][i + NW / 4];
                    v1 += acc[mh][i + 1 + NW / 4];
                  }
                  unsigned char* const e = row + (64 * mh + 8 * h) * 16;
                  if constexpr (TERMS == 1) {
                    *reinterpret_cast<uint32_t*>(e) = bf16_pair(leaky(v0 + b0, slope), leaky(v1 + b1, slope));
                  } else {
                    uint32_t hi, lo;
                    split_pair(leaky(v0 + b0, slope), leaky(v1 + b1, slope), hi, lo);
                    *reinterpret_cast<uint32_t*>(e) = hi;
                    *reinterpret_cast<uint32_t*>(e + MT * 16) = lo;
                  }
                }
            }
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            named_bar_sync(1 + r, 128);
            // first channel of row t = (group t / P, plane t % P)
            const int f = wk.nh * NCOL + pc * SCH + 8 * (t >> (P - 1));
            if (t < SCH * P / 8 && f < Cout) {
              const long long dst = sa::entry<P>(n, t & (P - 1), (xs.out_c0 + f) >> 3, (long long)y * OW + x0, xs.out_Cg,
                                                 oplane0);
              bulk_s2g(xs.out + dst, smem_u32(sst + t * MT * 16), seg * 4);
              bulk_commit();
            }
          }
        } else
#pragma unroll
        for (int pc = 0; pc < NCOL / SCH; ++pc) {
          if (t < SCH) bulk_wait_read();                  // this thread's previous copies have read the staging rows
          named_bar_sync(1 + r, 128);
#pragma unroll
          for (int jj = 0; jj < SCH / 8; ++jj) {
            const int j = pc * (SCH / 8) + jj;
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int f = wk.nh * NCOL + 8 * j + 2 * (lane & 3) + e;
              const float b = (bias != nullptr && f < Cout) ? __ldg(bias + f) : 0.f;
              const float sl = f < lin_prefix ? 1.f : slope;
              float* const row = stg + (8 * jj + 2 * (lane & 3) + e) * SPITCH + 16 * wq + (lane >> 2);
#pragma unroll
              for (int mh = 0; mh < MB; ++mh)
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                  const int i = 4 * j + 2 * h + e;
                  float v = acc[mh][i];
                  if constexpr (FOLD_ACC) v += acc[mh][i + NW / 4];
                  row[64 * mh + 8 * h] = leaky(v + b, sl);
                }
            }
          }
          asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy stores -> visible to the copy
          named_bar_sync(1 + r, 128);
          const int f = wk.nh * NCOL + pc * SCH + t;
          if (t < SCH && f < Cout) {
            bulk_s2g(out + (size_t)f * oplane0 + (size_t)y * OW + x0, smem_u32(stg + t * SPITCH), seg);
            bulk_commit();
          }
        }
      } else if (y < OH && !(dbg & 4)) {
#pragma unroll
        for (int mh = 0; mh < MB; ++mh) {
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int xx = tx * MT + 64 * mh + 16 * wq + (lane >> 2) + 8 * h;
            if (xx >= OW) continue;
#pragma unroll
            for (int j = 0; j < NCOL / 8; ++j) {
#pragma unroll
              for (int e = 0; e < 2; ++e) {
                const int i = 4 * j + 2 * h + e;
                float v = acc[mh][i];
                if constexpr (FOLD_ACC) v += acc[mh][i + NW / 4];   // second column block: the hi * lo term
                const int f = wk.nh * NCOL + 8 * j + 2 * (lane & 3) + e;
                if (f >= Cout) continue;
                if (xs.out != nullptr && !partial && f >= lin_prefix) {
                  // split output: the pair (f, f + 1) as one hi and one lo word (f - lin_prefix is even, host-checked)
                  if (e == 0) {
                    const float b0 = bias != nullptr ? __ldg(bias + f) : 0.f, b1 = bias != nullptr ? __ldg(bias + f + 1) : 0.f;
                    float v1 = acc[mh][i + 1];
                    if constexpr (FOLD_ACC) v1 += acc[mh][i + 1 + NW / 4];
                    sa::put_pair<P>(xs.out, xs.out_Cg, oplane0, n, xs.out_c0 + f - lin_prefix, (size_t)y * OW + xx,
                                 leaky(v + b0, slope), leaky(v1 + b1, slope));
                  }
                } else if (out_mode == 0) {
                  const float t = v + (bias != nullptr ? __ldg(bias + f) : 0.f);
                  out[(size_t)f * oplane0 + (size_t)y * OW + xx] = leaky(t, f < lin_prefix ? 1.f : slope);
                } else {
                  // depth-to-space: conv channel f = (2 py + px) * F + ff  ->  out[n][ff][2y + py][2x + px]
                  const int ph = f / F, ff = f - ph * F;
                  const float t = v + (bias != nullptr ? __ldg(bias + ff) : 0.f);
                  out[(size_t)ff * oplane2 + (size_t)(2 * y + (ph >> 1)) * (2 * OW) + 2 * xx + (ph & 1)] = leaky(t, slope);
                }
              }
            }
          }
        }
      }
    }
    bulk_wait_all();   // the staged epilogue's last copies have completed before the CTA (and its shared memory) ends
  } else if (warp == 8) {
    // ============================ weight loader (one thread) ============================
    if (lane == 0) {
      uint32_t ws = 0, wph = 0;
      bool wrapped = false;
      for (int work = blockIdx.x; work < numWork; work += gridDim.x) {
        const Work wk = decode_work(work, sk, nChunks);
        const int cb = wk.cb, ce = wk.ce;
        if constexpr (TERMS == 3) {
          const unsigned char* src = wpack + (size_t)cb * 9 * sm.w_tile;
          for (int it = 9 * cb; it < 9 * ce; it += TPS, src += sm.w_stage) {
            if (wrapped) mbar_wait(w_empty + 8 * ws, wph ^ 1);
            if (dbg & 32) {   // profiling: no weight copies, the stage holds whatever it held
              mbar_arrive(w_full + 8 * ws);
            } else {
              mbar_arrive_expect_tx(w_full + 8 * ws, (uint32_t)sm.w_stage);
              bulk_g2s(s_base + (uint32_t)sm.w_off + ws * (uint32_t)sm.w_stage, src, (uint32_t)sm.w_stage, w_full + 8 * ws);
            }
            if (++ws == (uint32_t)WS) { ws = 0; wph ^= 1; wrapped = true; }
          }
        } else {
          // the hi half of each tap's packed tile (64 CoutP bytes in global memory): one contiguous run, or -- folded
          // layout, [plane][hi rows | lo rows] -- one run of CoutP rows per 8-channel plane
          const int gt = 64 * CoutP, run = 16 * CoutP;
          const unsigned char* src = wpack + (size_t)cb * 9 * gt;
          for (int it = 9 * cb; it < 9 * ce; it += TPS, src += TPS * gt) {
            if (wrapped) mbar_wait(w_empty + 8 * ws, wph ^ 1);
            if (dbg & 32) {   // profiling: no weight copies
              mbar_arrive(w_full + 8 * ws);
              if (++ws == (uint32_t)WS) { ws = 0; wph ^= 1; wrapped = true; }
              continue;
            }
            mbar_arrive_expect_tx(w_full + 8 * ws, (uint32_t)sm.w_stage);
            const uint32_t dst = s_base + (uint32_t)sm.w_off + ws * (uint32_t)sm.w_stage;
#pragma unroll 1
            for (int t = 0; t < TPS; ++t) {
              if constexpr (FOLD) {
                bulk_g2s(dst + (uint32_t)(t * sm.w_tile), src + t * gt, (uint32_t)run, w_full + 8 * ws);
                bulk_g2s(dst + (uint32_t)(t * sm.w_tile + run), src + t * gt + 2 * run, (uint32_t)run, w_full + 8 * ws);
              } else {
                bulk_g2s(dst + (uint32_t)(t * sm.w_tile), src + t * gt, (uint32_t)sm.w_tile, w_full + 8 * ws);
              }
            }
            if (++ws == (uint32_t)WS) { ws = 0; wph ^= 1; wrapped = true; }
          }
        }
      }
    }
  } else {
    // ============================ input producers (warps 9..11) ============================
    if (xs.in == 1) {
      // split input (split_act.cuh): the buffer already holds the converted entries in the stage layout, and each image
      // row of one group and plane is one contiguous run of 16-byte entries.  So a chunk is nslots x 2 groups x P planes
      // 1-D bulk copies of the tile row's in-image pixels, one per lane of warp 9 (at most 6 x 2 x 2 = 24).  Each lane
      // first zeroes the entries of its row that lie outside the image (the padding; the stage may hold another tile's
      // data there).  (A tensor copy of the same box moves one 16-byte entry per box row: that delivered a stage about
      // as slowly as the MMAs of a narrow layer consume it.)
      if (warp == 9) {
        uint32_t as = 0, aph = 0;
        bool wrapped = false;
        const long long HW = (long long)H * W;
        const int ncp = nslots * 2 * P;
        const int pl = lane % P, kc = (lane / P) & 1, s = lane / (2 * P);   // this lane's row: plane, group, slot
        const bool mine = lane < ncp;
        const int ky = s / R, rr = s - ky * R;
        for (int work = blockIdx.x; work < numWork; work += gridDim.x) {
          const Work wk = decode_work(work, sk, nChunks);
          int tx, ty, n;
          decode_tile(wk.tile, tilesX, tilesY, sk, tx, ty, n);
          const int x0 = tx * MT - dil, y0 = ty * R;
          const int xa = x0 > 0 ? x0 : 0, xb = x0 + PW < W ? x0 + PW : W;
          const int e0 = xa - x0, e1 = xb - x0;                 // entries [e0, e1) of a row lie inside the image
          const int y = dil < R ? y0 - dil + s : y0 + (ky - 1) * dil + rr;
          const bool row_in = mine && (unsigned)y < (unsigned)H;
          const uint32_t bytes = (uint32_t)__popc(__ballot_sync(0xffffffffu, row_in)) * (uint32_t)(e1 - e0) * 16u;
          for (int c = wk.cb; c < wk.ce; ++c) {
            if (wrapped) mbar_wait(a_empty + 8 * as, aph ^ 1);
            const uint32_t bar = a_full + 8 * as;
            if (dbg & 16) {
              if (lane == 0) mbar_arrive(bar);
            } else {
              unsigned char* const row = smem + as * sm.a_stage + pl * sm.a_lo + (kc * E + s * PW) * 16;
              if (mine) {
                const int z0 = row_in ? e0 : PW;
                for (int e = 0; e < z0; ++e) *reinterpret_cast<uint4*>(row + e * 16) = make_uint4(0u, 0u, 0u, 0u);
                if (row_in)
                  for (int e = e1; e < PW; ++e) *reinterpret_cast<uint4*>(row + e * 16) = make_uint4(0u, 0u, 0u, 0u);
              }
              asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy zeros -> tensor core
              __syncwarp();
              if (lane == 0) mbar_arrive_expect_tx(bar, bytes);
              __syncwarp();
              if (row_in) {
                const long long src = sa::entry<P>(n, pl, xs.in_g0 + 2 * c + kc, (long long)y * W + xa, xs.in_Cg, HW);
                bulk_g2s(smem_u32(row + e0 * 16), xs.in_buf + src, (uint32_t)(e1 - e0) * 16u, bar);
              }
            }
            if (++as == (uint32_t)AS) { as = 0; aph ^= 1; wrapped = true; }
          }
        }
      }
      return;
    }
    // One instruction stream for every layer shape: the (work item, chunk, batch) space of this CTA is walked as ONE flat
    // sequence of batches (BATCH items of 32 entries x 8 channels per warp), software-pipelined over two register sets --
    // the loads of batch i+1 (possibly the next chunk, possibly the next TILE) are in flight while batch i is converted and
    // stored.  Geometry is arithmetic only (e / PW through a multiply-high).
    if (dbg & 16) {   // profiling: no input path at all -- the same a_empty / a_full traffic per chunk, nothing loaded or stored
      uint32_t as = 0, aph = 0;
      bool wrapped = false;
      for (int work = blockIdx.x; work < numWork; work += gridDim.x) {
        const Work wk = decode_work(work, sk, nChunks);
        for (int c = wk.cb; c < wk.ce; ++c) {
          if (wrapped) mbar_wait(a_empty + 8 * as, aph ^ 1);
          __syncwarp();
          if (lane == 0) mbar_arrive(a_full + 8 * as);
          if (++as == (uint32_t)AS) { as = 0; aph ^= 1; wrapped = true; }
        }
      }
      return;
    }
    const int pw = warp - 9;
    const int G = (E + 31) / 32;
    const bool one_plane = Cin <= 8;          // a single chunk whose channels 8..15 are zeros: plane 1 is cleared once, never loaded
    const int nItems = one_plane ? G : 2 * G;                        // item = (32 entries, 8-channel plane)
    const int nb = (nItems + NPROD * BATCH - 1) / (NPROD * BATCH);   // batches per stage (and warp)
    const uint32_t pw_magic = 0xFFFFFFFFu / (uint32_t)PW + 1u;       // e / PW == umulhi(e, magic)  (e * PW < 2^32)
    if (one_plane) {
      for (int st = 0; st < AS; ++st)
        for (int e = pw * 32 + lane; e < E; e += NPROD * 32) {
          unsigned char* d = smem + st * sm.a_stage + (E + e) * 16;
          *reinterpret_cast<uint4*>(d) = make_uint4(0u, 0u, 0u, 0u);
          if constexpr (P == 2) *reinterpret_cast<uint4*>(d + sm.a_lo) = make_uint4(0u, 0u, 0u, 0u);
        }
    }
    if (xs.in == 2) {
      // TMA-staged fp32 input (dilation 1): one thread copies each chunk's raw tile -- at stride 1 the box {MT + 8 pixels
      // from x0 - 4, the 4 rows from y0 - 1, 16 channels}, at stride 2 one box {2 MT + 4 pixels from 2 x0 - 4, the 5 rows
      // from 2 y0 - 1, 8 channels} per 8-channel plane (raw_pitch) of the tensor map {W, H, Cin, N}, out-of-bounds pixels,
      // rows and channels read zero: the padding -- into a ring of RS raw stages, RS stages ahead of the conversion and
      // across tile boundaries.  The producers convert from shared memory the same entries, in the same layout, as the
      // loads below.  Their per-element work is then a shared-memory load at a fixed offset: no geometry checks and no
      // address chains.
      const bool s2 = stride == 2;
      const int RP = raw_pitch(MT, stride), CP = nslots * RP;   // raw row and channel pitch, in floats
      const int RPC = s2 && !one_plane ? 2 : 1;                 // raw stages per chunk (Cin <= 8: plane 1 stays zero)
      const uint32_t raw_bytes = (uint32_t)sm.raw_stage, raw_base = s_base + (uint32_t)sm.raw_off;
      const bool issuer = warp == 9 && lane == 0;
      int i_work = blockIdx.x, i_c = 0, i_h = 0, i_ce = 0, i_x = 0, i_y = 0, i_n = 0;   // issue cursor
      auto i_tile = [&]() {
        if (i_work >= numWork) return;
        const Work wk = decode_work(i_work, sk, nChunks);
        int tx, ty;
        decode_tile(wk.tile, tilesX, tilesY, sk, tx, ty, i_n);
        i_c = wk.cb;
        i_ce = wk.ce;
        // a 16-byte aligned start: the inner box coordinate of a tensor copy must be
        i_x = s2 ? 2 * tx * MT - 4 : tx * MT - 4;
        i_y = s2 ? 2 * ty * R - 1 : ty * R - 1;
      };
      auto issue = [&](uint32_t slot) {   // the cursor's chunk (plane i_h at stride 2) into raw stage `slot`
        if (i_work >= numWork) return;
        const uint32_t bar = r_full + 8 * slot;
        if (dbg & 2) {   // profiling: no global loads, the stage converts whatever it holds
          mbar_arrive(bar);
        } else {
          mbar_arrive_expect_tx(bar, raw_bytes);
          tma_load_4d(raw_base + slot * raw_bytes, &tmx, i_x, i_y, 16 * i_c + 8 * i_h, i_n, bar);
        }
        if (++i_h < RPC) return;
        i_h = 0;
        if (++i_c >= i_ce) {
          i_work += gridDim.x;
          i_tile();
        }
      };
      if (issuer) {
        i_tile();
        for (int s = 0; s < RS; ++s) issue((uint32_t)s);
      }
      uint32_t as = 0, aph = 0, rs = 0, rph = 0;
      bool wrapped = false;
      for (int work = blockIdx.x; work < numWork; work += gridDim.x) {
        const Work wk = decode_work(work, sk, nChunks);
        for (int c = wk.cb; c < wk.ce; ++c) {
          unsigned char* a_st = smem + as * sm.a_stage;
          for (int h = 0; h < RPC; ++h) {
            mbar_wait(r_full + 8 * rs, rph);
            if (h == 0 && wrapped) mbar_wait(a_empty + 8 * as, aph ^ 1);   // the MMAs that read this stage have completed
            const float* raw = reinterpret_cast<const float*>(smem + sm.raw_off + rs * raw_bytes);
            auto put = [&](int kc, int e, const float (&v)[8]) {
              if constexpr (P == 1) {
                *reinterpret_cast<uint4*>(a_st + (kc * E + e) * 16) =
                    make_uint4(bf16_pair(v[0], v[1]), bf16_pair(v[2], v[3]), bf16_pair(v[4], v[5]), bf16_pair(v[6], v[7]));
              } else {
                uint4 hi, lo;
                split_pair(v[0], v[1], hi.x, lo.x);
                split_pair(v[2], v[3], hi.y, lo.y);
                split_pair(v[4], v[5], hi.z, lo.z);
                split_pair(v[6], v[7], hi.w, lo.w);
                unsigned char* dst = a_st + (kc * E + e) * 16;
                *reinterpret_cast<uint4*>(dst) = hi;
                *reinterpret_cast<uint4*>(dst + sm.a_lo) = lo;
              }
            };
            if (s2) {
              // plane h.  Unit j of row s reads the adjacent pair raw[c][s][2 j + 2 .. 2 j + 3] (one 8-byte load per
              // channel: consecutive lanes, consecutive words) and writes odd entry MT + j and even entry j - 1.
              constexpr int U = MT + 1;   // units per row
              for (int u = pw * 32 + lane; u < (2 * R + 1) * U; u += NPROD * 32) {
                const int slot = u / U, j = u - slot * U;
                const float* s = raw + slot * RP + 2 * j + 2;
                float ve[8], vo[8];
#pragma unroll
                for (int jj = 0; jj < 8; ++jj) {
                  const float2 p2 = *reinterpret_cast<const float2*>(s + jj * CP);
                  ve[jj] = p2.x;
                  vo[jj] = p2.y;
                }
                put(h, slot * PW + MT + j, vo);
                if (j > 0) put(h, slot * PW + j - 1, ve);
              }
            } else {
#pragma unroll 2
              for (int t = pw; t < nItems; t += NPROD) {
                const int kc = one_plane ? 0 : (t & 1);
                const int e = (one_plane ? t : (t >> 1)) * 32 + lane;
                if (e >= E) continue;
                const int slot = e / (MT + 2), pe = e - slot * (MT + 2);   // PW = MT + 2 at stride 1, dilation 1
                const float* s = raw + 8 * kc * CP + slot * RP + pe + 3;
                float v[8];
#pragma unroll
                for (int jj = 0; jj < 8; ++jj) v[jj] = s[jj * CP];
                put(kc, e, v);
              }
            }
            const bool last = h == RPC - 1;
            if (last) asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy stores -> tensor core
            __syncwarp();
            if (lane == 0) {
              if (last) mbar_arrive(a_full + 8 * as);
              mbar_arrive(r_empty + 8 * rs);   // this warp has read the raw stage
            }
            if (issuer) {   // all three have: refill it RS stages ahead
              mbar_wait(r_empty + 8 * rs, rph);
              issue(rs);
            }
            __syncwarp();
            if (++rs == (uint32_t)RS) { rs = 0; rph ^= 1; }
          }
          if (++as == (uint32_t)AS) { as = 0; aph ^= 1; wrapped = true; }
        }
      }
      return;
    }
    // load cursor (runs one batch ahead of the store cursor)
    int l_work = blockIdx.x, l_c = 0, l_kb = 0, l_x0 = 0, l_y0 = 0;
    const float* l_xn = x;
    int l_ce = nChunks;        // end of this work item's chunk range (split-K)
    auto set_tile = [&]() {
      const Work wk = decode_work(l_work, sk, nChunks);
      l_c = wk.cb;
      l_ce = wk.ce;
      int tx, ty, n;
      decode_tile(wk.tile, tilesX, tilesY, sk, tx, ty, n);
      // ext = 1: "full" convolution -- the output grid is the input grid extended by one pixel on every side
      // (OH = H + 2, OW = W + 2; output (y, x) sits at input position (y - 1, x - 1)); used by K3 through linearity
      l_x0 = tx * MT - (ext ? 1 : 0);
      l_y0 = ty * R - (ext ? 1 : 0);
      l_xn = x + (size_t)n * x_bs;
    };
    auto advance = [&]() {   // false when this CTA's sequence is exhausted
      if (++l_kb < nb) return true;
      l_kb = 0;
      if (++l_c < l_ce) return true;
      l_work += gridDim.x;
      if (l_work >= numWork) return false;
      set_tile();
      return true;
    };
    // Geometry without branches: y = ymul * y0 + ya + yb * (slot >> 1) + yc * (slot & 1) + yd * slot, x likewise (see
    // slot_of / tap_xoff); addresses = one uniform 64-bit chunk base + 32-bit element offsets (16 planes < 2^32
    // elements, checked by the host), so a load costs one add and one IMAD.WIDE instead of a 64-bit add chain.
    const bool s2 = stride == 2, wide = !s2 && dil >= R;
    const int ymul = s2 ? 2 : 1, ya = s2 ? -1 : -dil, yb = wide ? dil : 0, yc = wide ? 1 : 0, yd = wide ? 0 : 1;
    const int xa = s2 ? 0 : -dil;
    const uint32_t planeu = (uint32_t)plane;
    auto load_batch = [&](float (&v)[BATCH][8]) {
      const float* xc = l_xn + (size_t)(16 * l_c) * plane;   // warp-uniform
      const int ybase = ymul * l_y0 + ya, xbase = ymul * l_x0 + xa;
#pragma unroll
      for (int b = 0; b < BATCH; ++b) {
        const int t = pw + (l_kb * BATCH + b) * NPROD;
        const int kc = one_plane ? 0 : (t & 1);
        const int e = (one_plane ? t : (t >> 1)) * 32 + lane;
        const int slot = (int)__umulhi((uint32_t)e, pw_magic), pe = e - slot * PW;
        int y = ybase + yb * (slot >> 1) + yc * (slot & 1) + yd * slot;
        const int q = (s2 && pe >= MT) ? 1 : 0;              // stride 2: odd-pixel block of the de-interleaved row
        int xx = xbase + ymul * (pe - q * MT) - q;           // q = 1: 2 (x0 - 1 + pe - MT) + 1
        if (ext == 2) {
          y = y >= 0 ? band_map(y, H) : -1;
          xx = xx >= 0 ? band_map(xx, W) : -1;
        }
        const bool ok = t < nItems && e < E && (unsigned)y < (unsigned)H && (unsigned)xx < (unsigned)W && !(dbg & 2);
        const int c0 = 16 * l_c + 8 * kc;
        uint32_t off = (uint32_t)(8 * kc) * planeu + (ok ? (uint32_t)(y * W + xx) : 0u);
        if (c0 + 8 <= Cin) {
#pragma unroll
          for (int jj = 0; jj < 8; ++jj) {
            v[b][jj] = ok ? __ldg(xc + off) : 0.f;
            off += planeu;
          }
        } else {
#pragma unroll
          for (int jj = 0; jj < 8; ++jj) {
            v[b][jj] = (ok && c0 + jj < Cin) ? __ldg(xc + off) : 0.f;
            off += planeu;
          }
        }
      }
    };
    // store cursor: batch index inside the stage + the running position in the input ring
    uint32_t as = 0, aph = 0;
    bool wrapped = false;
    auto store_batch = [&](int kb, const float (&v)[BATCH][8]) {
      if (kb == 0 && wrapped) mbar_wait(a_empty + 8 * as, aph ^ 1);   // the MMAs that read this stage have completed
      unsigned char* a_st = smem + as * sm.a_stage;
#pragma unroll
      for (int b = 0; b < BATCH; ++b) {
        const int t = pw + (kb * BATCH + b) * NPROD;
        const int kc = one_plane ? 0 : (t & 1);
        const int e = (one_plane ? t : (t >> 1)) * 32 + lane;
        if (t < nItems && e < E) {
          if constexpr (P == 1) {
            *reinterpret_cast<uint4*>(a_st + (kc * E + e) * 16) = make_uint4(
                bf16_pair(v[b][0], v[b][1]), bf16_pair(v[b][2], v[b][3]), bf16_pair(v[b][4], v[b][5]), bf16_pair(v[b][6], v[b][7]));
          } else {
            uint4 hi, lo;
            split_pair(v[b][0], v[b][1], hi.x, lo.x);
            split_pair(v[b][2], v[b][3], hi.y, lo.y);
            split_pair(v[b][4], v[b][5], hi.z, lo.z);
            split_pair(v[b][6], v[b][7], hi.w, lo.w);
            unsigned char* dst = a_st + (kc * E + e) * 16;
            *reinterpret_cast<uint4*>(dst) = hi;
            *reinterpret_cast<uint4*>(dst + sm.a_lo) = lo;
          }
        }
      }
      if (kb == nb - 1) {
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy stores -> visible to the tensor core
        __syncwarp();
        if (lane == 0) mbar_arrive(a_full + 8 * as);
        if (++as == (uint32_t)AS) { as = 0; aph ^= 1; wrapped = true; }
      }
    };
    float va[BATCH][8], vb[BATCH][8];
    set_tile();
    load_batch(va);
    int s_kb = 0;
    for (;;) {
      bool more = advance();
      if (more) load_batch(vb);
      store_batch(s_kb, va);
      if (!more) break;
      s_kb = l_kb;
      more = advance();
      if (more) load_batch(va);
      store_batch(s_kb, vb);
      if (!more) break;
      s_kb = l_kb;
    }
  }
}

// ---------------------------------------------------------------------------------------------------------
long long conv3x3_wgmma_packed_bytes(int Cin, int Cout) {
  return (long long)((Cin + 15) / 16) * 9 * 64 * um::cout_pad(Cout);
}

int conv3x3_wgmma_pack(const float* weight, unsigned char* packed, int Cin, int Cout, cudaStream_t st) {
  const int CoutP = um::cout_pad(Cout), nChunks16 = (Cin + 15) / 16;
  const long long total = (long long)nChunks16 * 9 * CoutP * 8;
  long long blocks = (total + 255) / 256;
  if (blocks > 4096) blocks = 4096;
  conv3x3_pack_wgmma_kernel<<<(unsigned)blocks, 256, 0, st>>>(weight, packed, Cin, Cout, CoutP, nChunks16);
  return check_launch("conv3x3_pack_wgmma_kernel");
}

// Split-K second pass over the split region (samples n_lo.., rows y_lo..): out = act(sum_p parts[p] + bias), NCHW (with
// the linear prefix) or depth-to-space.  TERMS as in the main kernel: split outputs have 2 / TERMS planes.
template <int TERMS>
__global__ void conv3x3_wgmma_reduce_kernel(um::SplitK sk, um::SplitDev xs, int RN, const float* __restrict__ bias,
                                            float* __restrict__ out, long long out_bs, int Cout, int OH, int OW, float slope,
                                            int out_mode_arg) {
  const int out_mode = out_mode_arg & 0xff, lin_prefix = out_mode_arg >> 8;
  const long long total = (long long)RN * Cout * sk.rh * OW;
  const int F = Cout >> 2;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    float s = 0.f;
    for (int p = 0; p < sk.k; ++p) s += sk.ws[(size_t)p * (size_t)sk.part_stride + (size_t)i];
    const int x = (int)(i % OW), y = sk.y_lo + (int)((i / OW) % sk.rh), f = (int)((i / ((long long)OW * sk.rh)) % Cout);
    const int n = sk.n_lo + (int)(i / ((long long)OW * sk.rh * Cout));
    if (out_mode == 0) {
      const float b = bias ? __ldg(bias + f) : 0.f;
      const float v = leaky(s + b, f < lin_prefix ? 1.f : slope);
      if (xs.out != nullptr && f >= lin_prefix)
        sa::put_one<TERMS == 1 ? 1 : 2>(xs.out, xs.out_Cg, (long long)OH * OW, n, xs.out_c0 + f - lin_prefix, (long long)y * OW + x, v);
      else
        out[(size_t)n * out_bs + ((size_t)f * OH + y) * OW + x] = v;
    } else {
      const int ph = f / F, ff = f - ph * F;
      const float b = bias ? __ldg(bias + ff) : 0.f;
      out[(size_t)n * out_bs + ((size_t)ff * (2 * OH) + (2 * y + (ph >> 1))) * (2 * OW) + 2 * x + (ph & 1)] = leaky(s + b, slope);
    }
  }
}

// Split-K plan.  Two cases, both about tiles being indivisible units of a persistent grid of one CTA per SM:
//   small images (levels 5-6: 2 x tiles <= SMs, up to 43 chunks walked serially per tile): every tile is cut into k parts;
//   a short last round (e.g. level 2 at batch 6 on 132 SMs: 672 tiles = 5 x 132 + 12 -- the 12 left-over tiles would cost a
//     6th round): only the tail tiles are cut, into as many parts as there are idle SMs, so the last round shrinks to 1/k
//     of a tile.  The tail is kept inside the last sample and aligned to whole tile rows, so the split region is a row range.
// Returns k = 1 when nothing is split.
static um::SplitK plan_split(int N, int Cin, int H, int W, int Cout, int stride, int dil, int grid_cap) {
  using namespace um;
  (void)dil;
  const int ns = cout_pad(Cout) > 128 ? 2 : 1;
  SplitK sk = {1, 0, 0, 0, 0, 0, nullptr, 0u, 0u, 3, ns};
  const int OH = (H - 1) / stride + 1, OW = (W - 1) / stride + 1, nChunks = (Cin + 15) / 16;
  // the launch's tile width: OW <= 64 is one tile column in either geometry, so only stride 2 with OW > 64 depends on it
  const int MT = tile_width(OW, stride);
  const int tilesX = (OW + MT - 1) / MT, tilesY = (OH + R - 1) / R;
  const long long tiles = (long long)N * tilesX * tilesY;
  sk.from = (int)tiles;
  const int mode = tuning().conv_splitk;
  if (!mode || tiles >= (1 << 29)) return sk;
  const int sms = grid_cap > 0 && grid_cap < kNumSMs ? grid_cap : kNumSMs;
  const int kcap = mode > 1 ? mode : 32;
  if (2 * tiles * ns <= sms) {                  // small image: split every tile
    int k = (int)(sms / (tiles * ns));
    if (k > nChunks / 3) k = nChunks / 3;       // at least 3 chunks per part
    if (k > 8) k = 8;
    if (k > kcap) k = kcap;
    if (k >= 2) {
      sk.k = k; sk.from = 0; sk.n_lo = 0; sk.y_lo = 0; sk.rh = OH;
    }
  } else if (ns == 1 && tiles > sms) {          // short last round: split the tail
    const long long rounds = tiles / sms;
    long long tail = tiles - rounds * sms;
    tail = (tail + tilesX - 1) / tilesX * tilesX;                 // whole tile rows
    int k = tail > 0 ? (int)(sms / tail) : 0;
    if (k > nChunks / 2) k = nChunks / 2;       // at least 2 chunks per part
    if (k > kcap) k = kcap;
    // only the long, tensor-bound layers gain more than the second launch costs; layers with few chunks or Cout <= 64
    // do not
    if (tail > 0 && tail <= (long long)tilesX * tilesY && rounds <= 12 && k >= 2 && nChunks >= 16 && Cout > 64) {
      sk.k = k; sk.from = (int)(tiles - tail); sk.n_lo = N - 1;
      sk.y_lo = (int)((sk.from / tilesX) % tilesY) * R;
      sk.rh = OH - sk.y_lo;
    }
  }
  if (sk.k > 1) sk.part_stride = (long long)(N - sk.n_lo) * Cout * sk.rh * OW;
  return sk;
}

long long conv3x3_wgmma_workspace_bytes(int N, int Cin, int H, int W, int Cout, int stride, int dil) {
  const um::SplitK sk = plan_split(N, Cin, H, W, Cout, stride, dil, tuning().conv_grid_cap);
  return sk.k > 1 ? sk.k * sk.part_stride * 4 : 0;
}

// returns -1 when the shape does not fit this kernel (caller falls back to the mma.sync kernel; split operands have no
// fall-back)
int conv3x3_wgmma_launch(const float* x, long long x_bs, const unsigned char* wpack, const float* bias, float* out,
                         long long out_bs, int N, int Cin, int H, int W, int Cout, int stride, int dil, int out_mode,
                         float slope, cudaStream_t st, int ext, float* ws, long long ws_bytes, const SplitIO& sio) {
  using namespace um;
  const int terms = (out_mode & MFN_CONV_BF16) ? 1 : 3;   // products per multiply-add; split operands have 2 / 1 planes
  out_mode &= ~MFN_CONV_BF16;
  const int grow = ext == 2 ? 8 : 2 * ext;   // ext 1: grid + 1 pixel per side; ext 2: + the six band rows / columns too
  const int OH = stride == 2 ? (H - 1) / 2 + 1 : H + grow, OW = stride == 2 ? (W - 1) / 2 + 1 : W + grow;
  const int MT = tile_width(OW, stride);
  SplitDev xs = {0, 0, 0, nullptr, nullptr, 0, 0};
  CUtensorMap tmx;
  memset(&tmx, 0, sizeof tmx);
  if (sio.in != nullptr) {
    // the row copies need 16-byte aligned rows, which every split buffer has; odd dilations >= R are not supported
    // (no layer has one)
    if (stride != 1 || ext != 0 || sio.in_c0 % 16 != 0 || (dil >= R && dil % 2 != 0) || !aligned(sio.in, 16)) return -1;
    xs.in = 1;
    xs.in_buf = static_cast<const unsigned char*>(sio.in);
    xs.in_g0 = sio.in_c0 / 8;
    xs.in_Cg = sa::groups(sio.in_C);
  }
  if (sio.out != nullptr) {
    // whole 16-channel chunks after the prefix: pairs stay pairs, and the buffer's pad channels are never written
    const int lp = out_mode >> 8;
    if ((out_mode & 0xff) != 0 || ext != 0 || sio.out_c0 % 16 != 0 || (Cout - lp) % 16 != 0 || lp % 2 != 0 ||
        sio.out_c0 + Cout - lp > sio.out_C || !aligned(sio.out, 16))
      return -1;
    xs.out = static_cast<unsigned char*>(sio.out);
    xs.out_Cg = sa::groups(sio.out_C);
    xs.out_c0 = sio.out_c0;
  }
  if (Cout > 256 || (stride != 1 && !(stride == 2 && dil == 1))) return -1;
  if (ext != 0 && !((ext == 1 || ext == 2) && stride == 1 && dil == 1 && out_mode == 0)) return -1;
  if ((out_mode >> 8) != 0 && (out_mode & 0xff) != 0) return -1;   // linear prefix only with plain NCHW output
  const int CoutP = um::cout_pad(Cout), nChunks = (Cin + 15) / 16;
  const int E = n_slots(stride, dil) * row_pitch(MT, stride, dil);
  const int as_wide = 3;   // input stages of the wide layers (smem_map)
  // staged epilogue (bulk copies of whole output row segments): plain NCHW output whose rows start 16-byte aligned
  // (split output: every row segment is 16-byte aligned; the register epilogue takes the linear prefix)
  const bool staged = (out_mode & 0xff) == 0 && ext == 0 &&
                      (xs.out != nullptr ? (out_mode >> 8) == 0 : OW % 4 == 0 && out_bs % 4 == 0 && aligned(out, 16)) &&
                      smem_map(E, CoutP, as_wide, STG_BYTES, terms).WS >= 2;
  // fp32 input staged raw by TMA (tuning "conv_tma_in"): dilation 1, no ext, stride 1 on 128-pixel tiles or stride 2 on
  // the 64-pixel tiles of outputs wider than 64 pixels, and a tensor map the hardware accepts -- a 16-byte aligned base and
  // 16-byte multiples for the row, plane and sample strides (W and x_bs multiples of 4) -- with room for the raw ring
  // beside at least 3 weight stages.  Everything else keeps the per-thread loads.  The tiles of outputs at most 64 pixels
  // wide (levels 4-6: few tiles, many chunks each) measured no faster with the raw ring at stride 1, whose two input
  // stages and shallower weight ring lengthen their serial chunk loop; their stride-2 layers are not measured with it.
  int raw = 0;
  const bool raw_geometry = stride == 1 ? dil == 1 && MT == MT_WIDE : MT == MT_NARROW && OW > MT_NARROW;
  if (sio.in == nullptr && tuning().conv_tma_in && raw_geometry && ext == 0 && W % 4 == 0 && x_bs % 4 == 0 &&
      aligned(x, 16)) {
    raw = raw_stage_bytes(n_slots(stride, 1), MT, stride);
    if (smem_map(E, CoutP, as_wide, staged ? STG_BYTES : 0, terms, raw, raw_ring_max(stride)).WS < 3) raw = 0;
  }
  if (raw) {
    EncodeTiledFn fn = encode_tiled_fn();
    if (fn == nullptr) return fail(MFN_ERR_UNSUPPORTED, "cuTensorMapEncodeTiled is not available from this driver");
    const cuuint64_t dim[4] = {(cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)Cin, (cuuint64_t)N};
    const cuuint64_t strides[3] = {(cuuint64_t)W * 4, (cuuint64_t)W * H * 4, (cuuint64_t)x_bs * 4};
    const cuuint32_t box[4] = {(cuuint32_t)raw_pitch(MT, stride), (cuuint32_t)n_slots(stride, 1),
                               (cuuint32_t)raw_channels(stride), 1};
    const cuuint32_t es[4] = {1, 1, 1, 1};
    const CUresult r = fn(&tmx, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, const_cast<float*>(x), dim, strides, box, es,
                          CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                          CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return fail(MFN_ERR_UNSUPPORTED, "cuTensorMapEncodeTiled failed (CUresult %d)", (int)r);
    xs.in = 2;
  }
  const SmemMap sm = smem_map(E, CoutP, as_wide, staged ? STG_BYTES : 0, terms, raw, raw_ring_max(stride));
  if (sm.WS < 2 || E * 16 > 0x3FFF * 16) return -1;
  if ((long long)H * W >= (1LL << 27)) return -1;   // the producers address a 16-plane chunk with 32-bit element offsets
  const int tilesX = (OW + MT - 1) / MT, tilesY = (OH + R - 1) / R;
  // split-K when the caller lent a workspace (plain grids only): one launch covers the whole tiles (normal epilogue) and the
  // parts of the split tiles (raw sums into the workspace), a second one reduces the split region
  const int ns = CoutP > 128 ? 2 : 1;
  SplitK sk = {1, 0, 0, 0, 0, 0, nullptr, 0u, 0u, 3, ns};
  if (ws != nullptr && ext == 0) {
    sk = plan_split(N, Cin, H, W, Cout, stride, dil, tuning().conv_grid_cap);
    if (sk.k > 1 && ws_bytes < sk.k * sk.part_stride * 4) sk.k = 1;
    sk.ws = ws;
  }
  const long long tiles = (long long)N * tilesX * tilesY;
  if (tiles * ns >= (1LL << 30)) return -1;
  sk.as_wide = as_wide;
  sk.stg = staged ? STG_BYTES : 0;
  if (sk.k <= 1) sk.from = (int)tiles;
  {
    const unsigned long long tp = (unsigned long long)tilesX * tilesY;
    if ((unsigned long long)tiles * tp < (1ull << 32) && tp * tilesX < (1ull << 32)) {   // q = umulhi(t, ceil(2^32 / d)) exact for t d < 2^32
      sk.magic_tp = (uint32_t)(((1ull << 32) + tp - 1) / tp);
      sk.magic_tx = tilesX == 1 ? 0u : (uint32_t)(((1ull << 32) + tilesX - 1) / tilesX);
    }
    if (tp == 1) sk.magic_tp = 0;          // ceil(2^32 / 1) does not fit 32 bits: the kernel divides
  }
  const long long numWork = (sk.from + (tiles - sk.from) * sk.k) * ns;
  const int cap = tuning().conv_grid_cap > 0 ? tuning().conv_grid_cap : kNumSMs;
  const unsigned grid = (unsigned)(numWork < cap ? numWork : cap);
  // variant name (last_kernel): the padded output width, whether the hi / lo weight images are folded, and bf16 for the
  // one-product variant (whose accumulator is CoutP wide in every layout).  Both tile widths, and both fp32 input paths
  // (per-thread loads or TMA-staged), share a name: they compute the same sums in the same order.
  const char* name = terms == 3 ? "conv3x3_wgmma_kernel<CoutP=256>" : "conv3x3_wgmma_kernel<CoutP=256,bf16>";
  // one instantiation set per tile width (mt: std::integral_constant); returns a CUDA error of the shared-memory opt-in
  auto launch = [&](auto mt) -> cudaError_t {
    constexpr int M = decltype(mt)::value;
    static SmemOptIn opt[8], opt1[8];
    cudaError_t e = cudaSuccess;
    if (terms == 3) {
      e = ensure_dyn_smem(conv3x3_wgmma_kernel<32, true, 9, 3, M>, sm.total, opt[0]);
      if (e == cudaSuccess) e = ensure_dyn_smem(conv3x3_wgmma_kernel<64, true, 9, 3, M>, sm.total, opt[1]);
      if (e == cudaSuccess) e = ensure_dyn_smem(conv3x3_wgmma_kernel<96, true, 3, 3, M>, sm.total, opt[2]);
      if (e == cudaSuccess) e = ensure_dyn_smem(conv3x3_wgmma_kernel<128, true, 3, 3, M>, sm.total, opt[3]);
      if (e == cudaSuccess) e = ensure_dyn_smem(conv3x3_wgmma_kernel<80, false, 1, 3, M>, sm.total, opt[4]);
      if (e == cudaSuccess) e = ensure_dyn_smem(conv3x3_wgmma_kernel<96, false, 1, 3, M>, sm.total, opt[5]);
      if (e == cudaSuccess) e = ensure_dyn_smem(conv3x3_wgmma_kernel<112, false, 1, 3, M>, sm.total, opt[6]);
      if (e == cudaSuccess) e = ensure_dyn_smem(conv3x3_wgmma_kernel<128, false, 1, 3, M>, sm.total, opt[7]);
    } else {
      e = ensure_dyn_smem(conv3x3_wgmma_kernel<16, true, 9, 1, M>, sm.total, opt1[0]);
      if (e == cudaSuccess) e = ensure_dyn_smem(conv3x3_wgmma_kernel<32, true, 9, 1, M>, sm.total, opt1[1]);
      if (e == cudaSuccess) e = ensure_dyn_smem(conv3x3_wgmma_kernel<48, true, 3, 1, M>, sm.total, opt1[2]);
      if (e == cudaSuccess) e = ensure_dyn_smem(conv3x3_wgmma_kernel<64, true, 3, 1, M>, sm.total, opt1[3]);
      if (e == cudaSuccess) e = ensure_dyn_smem(conv3x3_wgmma_kernel<80, false, 1, 1, M>, sm.total, opt1[4]);
      if (e == cudaSuccess) e = ensure_dyn_smem(conv3x3_wgmma_kernel<96, false, 1, 1, M>, sm.total, opt1[5]);
      if (e == cudaSuccess) e = ensure_dyn_smem(conv3x3_wgmma_kernel<112, false, 1, 1, M>, sm.total, opt1[6]);
      if (e == cudaSuccess) e = ensure_dyn_smem(conv3x3_wgmma_kernel<128, false, 1, 1, M>, sm.total, opt1[7]);
    }
    if (e != cudaSuccess) return e;
#define MFN_WGMMA_LAUNCH(NW_, FOLD_, TPS_, TERMS_)                                                                      \
  conv3x3_wgmma_kernel<NW_, FOLD_, TPS_, TERMS_, M><<<grid, NTHREADS, sm.total, st>>>(                                 \
      x, x_bs, wpack, bias, out, out_bs, Cin, H, W, OH, OW, Cout, CoutP, nChunks, slope, tilesX, tilesY, (int)numWork, \
      stride, dil, out_mode, ext, sk, xs, tmx, tuning().conv_dbg)
    if (terms == 3) {
      switch (CoutP) {
        case 16: MFN_WGMMA_LAUNCH(32, true, 9, 3); name = "conv3x3_wgmma_kernel<CoutP=16,fold>"; break;
        case 32: MFN_WGMMA_LAUNCH(64, true, 9, 3); name = "conv3x3_wgmma_kernel<CoutP=32,fold>"; break;
        case 48: MFN_WGMMA_LAUNCH(96, true, 3, 3); name = "conv3x3_wgmma_kernel<CoutP=48,fold>"; break;
        case 64: MFN_WGMMA_LAUNCH(128, true, 3, 3); name = "conv3x3_wgmma_kernel<CoutP=64,fold>"; break;
        case 80: MFN_WGMMA_LAUNCH(80, false, 1, 3); name = "conv3x3_wgmma_kernel<CoutP=80>"; break;
        case 96: MFN_WGMMA_LAUNCH(96, false, 1, 3); name = "conv3x3_wgmma_kernel<CoutP=96>"; break;
        case 112: MFN_WGMMA_LAUNCH(112, false, 1, 3); name = "conv3x3_wgmma_kernel<CoutP=112>"; break;
        case 128: MFN_WGMMA_LAUNCH(128, false, 1, 3); name = "conv3x3_wgmma_kernel<CoutP=128>"; break;
        default: MFN_WGMMA_LAUNCH(128, false, 1, 3);   // 256: two 128-channel halves per tile
      }
    } else {
      switch (CoutP) {
        case 16: MFN_WGMMA_LAUNCH(16, true, 9, 1); name = "conv3x3_wgmma_kernel<CoutP=16,fold,bf16>"; break;
        case 32: MFN_WGMMA_LAUNCH(32, true, 9, 1); name = "conv3x3_wgmma_kernel<CoutP=32,fold,bf16>"; break;
        case 48: MFN_WGMMA_LAUNCH(48, true, 3, 1); name = "conv3x3_wgmma_kernel<CoutP=48,fold,bf16>"; break;
        case 64: MFN_WGMMA_LAUNCH(64, true, 3, 1); name = "conv3x3_wgmma_kernel<CoutP=64,fold,bf16>"; break;
        case 80: MFN_WGMMA_LAUNCH(80, false, 1, 1); name = "conv3x3_wgmma_kernel<CoutP=80,bf16>"; break;
        case 96: MFN_WGMMA_LAUNCH(96, false, 1, 1); name = "conv3x3_wgmma_kernel<CoutP=96,bf16>"; break;
        case 112: MFN_WGMMA_LAUNCH(112, false, 1, 1); name = "conv3x3_wgmma_kernel<CoutP=112,bf16>"; break;
        case 128: MFN_WGMMA_LAUNCH(128, false, 1, 1); name = "conv3x3_wgmma_kernel<CoutP=128,bf16>"; break;
        default: MFN_WGMMA_LAUNCH(128, false, 1, 1);
      }
    }
#undef MFN_WGMMA_LAUNCH
    return cudaSuccess;
  };
  const cudaError_t e = MT == MT_NARROW ? launch(std::integral_constant<int, MT_NARROW>{})
                                        : launch(std::integral_constant<int, MT_WIDE>{});
  if (e != cudaSuccess) return fail((int)e, "cudaFuncSetAttribute(conv3x3_wgmma_kernel): %s", cudaGetErrorString(e));
  const int rc = check_launch(name);
  if (rc != 0 || sk.k <= 1) return rc;
  const long long total = sk.part_stride;
  long long blocks = (total + 255) / 256;
  if (blocks > 4 * kNumSMs) blocks = 4 * kNumSMs;
  if (terms == 3) {
    conv3x3_wgmma_reduce_kernel<3><<<(unsigned)blocks, 256, 0, st>>>(sk, xs, N - sk.n_lo, bias, out, out_bs, Cout, OH, OW, slope, out_mode);
    return check_launch("conv3x3_wgmma_reduce_kernel");
  }
  conv3x3_wgmma_reduce_kernel<1><<<(unsigned)blocks, 256, 0, st>>>(sk, xs, N - sk.n_lo, bias, out, out_bs, Cout, OH, OW, slope, out_mode);
  return check_launch("conv3x3_wgmma_reduce_kernel<bf16>");
}

}  // namespace mfn
