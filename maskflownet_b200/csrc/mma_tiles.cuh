// mma_tiles.cuh -- shared building blocks of the tensor-core implicit-GEMM kernels (conv3x3.cu, warp_mma.cu):
// bf16 hi/lo split, ldmatrix / mma.sync / cp.async wrappers, the XOR-swizzled 64-byte-per-row tile addressing and the
// packed-weight tile geometry.
#pragma once
#include <cuda_bf16.h>

#include "common.cuh"

namespace mfn {
namespace c3 {
constexpr int TW = 32, HX = 4, HWP = TW + 2 * HX;   // 40-pixel tile rows (quad aligned like the correlation tiles)
constexpr int PXB = 64;                              // bytes per pixel / per weight row: 32 channels bf16
constexpr int NTHREADS = 256;
constexpr int WSTAGES = 3;

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void split_pair(float a, float b, uint32_t& hi, uint32_t& lo) {
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(hi) : "f"(b), "f"(a));
  const float ah = __uint_as_float(hi << 16), bh = __uint_as_float(hi & 0xffff0000u);
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(lo) : "f"(b - bh), "f"(a - ah));
}
__device__ __forceinline__ void ldsm_x4(uint32_t addr, uint32_t (&r)[4]) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(addr)
               : "memory");
}
__device__ __forceinline__ void mma_bf16(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }
// byte offset of 16-byte chunk c (8 channels) of row p (pixel or output channel) inside a 64-byte-per-row buffer
__host__ __device__ __forceinline__ int swz(int p, int c) { return p * PXB + ((c ^ ((p >> 1) & 3)) << 4); }

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
