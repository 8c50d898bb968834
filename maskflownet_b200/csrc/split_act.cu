// split_act.cu -- fp32 NCHW channels -> a channel slice of a split-activation (or bf16-activation) buffer (split_act.cuh): the dense blocks'
// inputs (correlation, features, flow) enter the split buffer here, once, instead of being converted by every reader.
// The kernel also builds for the host (MFN_HOST_EMULATION: tests/host_emu/split_act_emu.cpp), one thread at a time.
#ifdef MFN_HOST_EMULATION
#include "cuda_shim.h"
#else
#include "common.cuh"
#endif
#include "split_act.cuh"

namespace mfn {

// one thread per (sample, 8-channel group of the slice, pixel): 8 coalesced fp32 loads -> one hi and one lo entry (P = 2),
// or one bf16 entry (P = 1: a bf16 activation); channels past C (up to the slice's 16-channel boundary) are written as
// zeros
template <int P = 2>
__global__ void split_pack_kernel(const float* __restrict__ src, long long src_bs, int C, unsigned char* __restrict__ dst,
                                  int dst_Cg, int g0, int N, long long HW) {
  const int G = sa::groups(C);
  const long long total = (long long)N * G * HW;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long p = i % HW;
    const int g = (int)((i / HW) % G), n = (int)(i / (HW * G));
    const float* s = src + (size_t)n * src_bs + (size_t)(8 * g) * HW + p;
    float v[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] = 8 * g + j < C ? __ldg(s + (size_t)j * HW) : 0.f;
    if constexpr (P == 1) {
      uint4 hi;
      hi.x = bf16_pair(v[0], v[1]);
      hi.y = bf16_pair(v[2], v[3]);
      hi.z = bf16_pair(v[4], v[5]);
      hi.w = bf16_pair(v[6], v[7]);
      *reinterpret_cast<uint4*>(dst + sa::entry<1>(n, 0, g0 + g, p, dst_Cg, HW)) = hi;
    } else {
      uint4 hi, lo;
      split_pair(v[0], v[1], hi.x, lo.x);
      split_pair(v[2], v[3], hi.y, lo.y);
      split_pair(v[4], v[5], hi.z, lo.z);
      split_pair(v[6], v[7], hi.w, lo.w);
      *reinterpret_cast<uint4*>(dst + sa::entry(n, 0, g0 + g, p, dst_Cg, HW)) = hi;
      *reinterpret_cast<uint4*>(dst + sa::entry(n, 1, g0 + g, p, dst_Cg, HW)) = lo;
    }
  }
}

}  // namespace mfn

#ifndef MFN_HOST_EMULATION
template <int P>
static int pack_slice(const char* fn, const float* src, long long src_batch_stride, int N, int C, int H, int W, void* dst,
                      int dst_channels, int dst_c0, void* stream) {
  using namespace mfn;
  MFN_REQUIRE(src && dst, MFN_ERR_INVALID_ARG, "%s: null pointer", fn);
  MFN_REQUIRE(N > 0 && C > 0 && H > 0 && W > 0, MFN_ERR_INVALID_ARG, "%s: non-positive extent", fn);
  MFN_REQUIRE(aligned(dst, 16), MFN_ERR_ALIGNMENT, "%s: destination buffer must be 16-byte aligned", fn);
  // the pad channels up to the slice's 16-channel boundary are written as zeros: they must be the buffer's own pad
  MFN_REQUIRE(dst_c0 >= 0 && dst_c0 % 16 == 0 && dst_c0 + C <= dst_channels &&
                  ((dst_c0 + C) % 16 == 0 || dst_c0 + C == dst_channels),
              MFN_ERR_INVALID_ARG,
              "%s: slice [%d, %d) of the %d channels must start at a multiple of 16 and end at one or at the last channel",
              fn, dst_c0, dst_c0 + C, dst_channels);
  const long long HW = (long long)H * W;
  const long long sbs = src_batch_stride ? src_batch_stride : (long long)C * HW;
  MFN_REQUIRE(sbs >= (long long)C * HW, MFN_ERR_INVALID_ARG, "%s: batch stride smaller than the tensor", fn);
  const long long total = (long long)N * sa::groups(C) * HW;
  long long blocks = (total + 255) / 256;
  if (blocks > 16 * kNumSMs) blocks = 16 * kNumSMs;
  split_pack_kernel<P><<<(unsigned)blocks, 256, 0, as_stream(stream)>>>(src, sbs, C, static_cast<unsigned char*>(dst),
                                                                       sa::groups(dst_channels), dst_c0 / 8, N, HW);
  return check_launch(P == 1 ? "split_pack_kernel<bf16>" : "split_pack_kernel");
}

extern "C" int mfn_split_pack(const float* src, long long src_batch_stride, int N, int C, int H, int W, void* dst,
                              int dst_channels, int dst_c0, void* stream) {
  return pack_slice<2>("mfn_split_pack", src, src_batch_stride, N, C, H, W, dst, dst_channels, dst_c0, stream);
}

extern "C" int mfn_bf16_pack(const float* src, long long src_batch_stride, int N, int C, int H, int W, void* dst,
                             int dst_channels, int dst_c0, void* stream) {
  return pack_slice<1>("mfn_bf16_pack", src, src_batch_stride, N, C, H, W, dst, dst_channels, dst_c0, stream);
}
#endif  // !MFN_HOST_EMULATION
