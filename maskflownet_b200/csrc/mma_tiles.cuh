// mma_tiles.cuh -- shared building blocks of the tensor-core implicit-GEMM kernels (conv3x3.cu, warp_mma.cu): the tile
// geometry of the mma.sync convolution and its packed weights (the PTX primitives are in ptx.cuh), and the entry points of
// the wgmma convolution.
#pragma once
#include <cuda_bf16.h>

#include "common.cuh"
#include "ptx.cuh"

namespace mfn {
namespace c3 {
constexpr int TW = 32, HX = 4, HWP = TW + 2 * HX;   // 40-pixel tile rows (quad aligned like the correlation tiles)
constexpr int PXB = 64;                              // bytes per pixel / per weight row: 32 channels bf16
constexpr int NTHREADS = 256;
constexpr int WSTAGES = 3;

// output channels padded to what the chosen warp layout covers (32 / 64 / 96 / 128): tiles never read outside the weight image
__host__ __device__ constexpr int cout_pad(int cout) { return cout <= 32 ? 32 : (cout <= 64 ? 64 : (cout <= 96 ? 96 : 128)); }
}  // namespace c3

// wgmma implementation of the same convolution (conv3x3_wgmma.cu); its weight image follows the mma.sync image
// inside the packed buffer.  conv3x3_wgmma_launch returns -1 when the shape does not fit (caller falls back).
long long conv3x3_sync_packed_bytes(int Cin, int Cout);
long long conv3x3_wgmma_packed_bytes(int Cin, int Cout);
int conv3x3_wgmma_pack(const float* weight, unsigned char* packed, int Cin, int Cout, cudaStream_t st);
// Split-activation operands (split_act.cuh) of one launch.  in != null: the input is channels [in_c0, in_c0 + Cin) of a
// split buffer of in_C channels (x is unused).  out != null: the output channels past the linear prefix go to channels
// out_c0.. of a split buffer of out_C channels; the prefix channels go to the fp32 `out` of the launch.
struct SplitIO {
  const void* in = nullptr;
  int in_C = 0, in_c0 = 0;
  void* out = nullptr;
  int out_C = 0, out_c0 = 0;
};
int conv3x3_wgmma_launch(const float* x, long long x_bs, const unsigned char* wpack, const float* bias, float* out,
                        long long out_bs, int N, int Cin, int H, int W, int Cout, int stride, int dil, int out_mode,
                        float slope, cudaStream_t st, int ext = 0, float* ws = nullptr, long long ws_bytes = 0,
                        const SplitIO& sio = SplitIO());
// cuTensorMapEncodeTiled through the runtime's driver entry point (no link against libcuda); null when unavailable
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn encode_tiled_fn();
// split-K over the input-channel chunks for layers with fewer tiles than SMs: the plan (1 = none) and the fp32 workspace
// the caller has to lend to conv3x3_wgmma_launch for it
long long conv3x3_wgmma_workspace_bytes(int N, int Cin, int H, int W, int Cout, int stride, int dil);

}  // namespace mfn
