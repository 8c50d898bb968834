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
int conv3x3_wgmma_launch(const float* x, long long x_bs, const unsigned char* wpack, const float* bias, float* out,
                        long long out_bs, int N, int Cin, int H, int W, int Cout, int stride, int dil, int out_mode,
                        float slope, cudaStream_t st, int ext = 0, float* ws = nullptr, long long ws_bytes = 0);
// split-K over the input-channel chunks for layers with fewer tiles than SMs: the plan (1 = none) and the fp32 workspace
// the caller has to lend to conv3x3_wgmma_launch for it
long long conv3x3_wgmma_workspace_bytes(int N, int Cin, int H, int W, int Cout, int stride, int dil);

}  // namespace mfn
