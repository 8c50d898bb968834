// split_act.cuh -- the split-activation format: an activation tensor stored already converted into the operands the wgmma
// convolution multiplies (the bf16 hi/lo split of bf16_split.cuh), in the layout its input tiles have in shared memory.
//
// A buffer of C channels holds Cg = ceil(C / 16) * 2 groups of 8 channels as (N, 2, Cg, H, W, 8) bf16: per sample first the
// hi image of every group, then the lo image; one 16-byte entry per (plane, group, pixel).  4 bytes per channel-pixel, as
// fp32.  Channels C .. 16 ceil(C / 16) - 1 are ZERO (the packed weights are zero there too, and 0 * NaN would poison the
// sum).  The convolution loads an input chunk (two groups, hi and lo) of a box of rows with one bulk copy per row, and the
// value it multiplies is bit for bit the split_pair of the fp32 value, so results do not depend on the input's format.
// Writers: the pack kernel (split_act.cu) and the wgmma convolution's epilogues, all through `entry` and split_pair;
// ops.SplitAct is the only Python code that knows the layout.
// A bf16 activation (the opt-in bf16 mode, MFN_CONV_BF16) is the same layout with P = 1 plane, (N, 1, Cg, H, W, 8): the hi
// image alone, each value rounded once to bf16 (bf16_pair), 2 bytes per channel-pixel.  The helpers take the plane count
// P as a template argument (2 = split, 1 = bf16).
#pragma once
#include "bf16_split.cuh"

namespace mfn {
namespace sa {
__host__ __device__ inline int groups(int C) { return (C + 15) / 16 * 2; }
// bytes of one sample
__host__ __device__ inline long long sample_bytes(int C, long long HW) { return 2LL * groups(C) * HW * 16; }
// byte offset of the 16-byte entry (sample n, plane 0 = hi / 1 = lo, group g, pixel p) of a buffer of Cg groups
template <int P = 2>
__host__ __device__ inline long long entry(int n, int plane, int g, long long p, int Cg, long long HW) {
  return (((long long)(P * n + plane) * Cg + g) * HW + p) * 16;
}
// channels (c, c + 1), c even, of pixel p
template <int P = 2>
__device__ __forceinline__ void put_pair(unsigned char* buf, int Cg, long long HW, int n, int c, long long p, float a, float b) {
  if constexpr (P == 1) {
    *reinterpret_cast<uint32_t*>(buf + entry<P>(n, 0, c >> 3, p, Cg, HW) + (c & 7) * 2) = bf16_pair(a, b);
  } else {
    uint32_t hi, lo;
    split_pair(a, b, hi, lo);
    unsigned char* e = buf + entry<P>(n, 0, c >> 3, p, Cg, HW) + (c & 7) * 2;
    *reinterpret_cast<uint32_t*>(e) = hi;
    *reinterpret_cast<uint32_t*>(e + (long long)Cg * HW * 16) = lo;
  }
}
// channel c of pixel p
template <int P = 2>
__device__ __forceinline__ void put_one(unsigned char* buf, int Cg, long long HW, int n, int c, long long p, float v) {
  if constexpr (P == 1) {
    *reinterpret_cast<uint16_t*>(buf + entry<P>(n, 0, c >> 3, p, Cg, HW) + (c & 7) * 2) = (uint16_t)bf16_pair(v, 0.f);
  } else {
    uint32_t hi, lo;
    split_pair(v, 0.f, hi, lo);
    unsigned char* e = buf + entry<P>(n, 0, c >> 3, p, Cg, HW) + (c & 7) * 2;
    *reinterpret_cast<uint16_t*>(e) = (uint16_t)hi;
    *reinterpret_cast<uint16_t*>(e + (long long)Cg * HW * 16) = (uint16_t)lo;
  }
}
}  // namespace sa
}  // namespace mfn
