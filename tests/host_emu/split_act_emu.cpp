// split_act_emu.cpp -- TEST INFRASTRUCTURE ONLY.  Compiles the split-activation pack kernel (maskflownet_b200/csrc/
// split_act.cu) for the host through cuda_shim.h and runs it thread by thread; C ABI for tests/test_split_act_host.py.
//   g++ -O1 -ffp-contract=off -shared -fPIC -I tests/host_emu split_act_emu.cpp
#define MFN_HOST_EMULATION 1
#include <cstring>

#include "cuda_shim.h"

// what the kernel uses beyond the shim: the vector type, the bit cast, and the one PTX instruction of the split,
// cvt.rn.bf16x2.f32 -- round to nearest even, NaN to the canonical bf16 NaN
struct uint4 {
  unsigned x, y, z, w;
};
static inline float __uint_as_float(unsigned u) {
  float f;
  std::memcpy(&f, &u, sizeof f);
  return f;
}
namespace mfn {
static inline uint32_t bf16_rn_(float f) {
  uint32_t u;
  std::memcpy(&u, &f, sizeof u);
  if ((u & 0x7fffffffu) > 0x7f800000u) return 0x7fffu;
  return (u + 0x7fffu + ((u >> 16) & 1u)) >> 16;
}
static inline uint32_t cvt_bf16x2_rn(float first, float second) { return bf16_rn_(first) | (bf16_rn_(second) << 16); }
}  // namespace mfn

#include "../../maskflownet_b200/csrc/split_act.cu"

using namespace mfn;

#define EMU_API extern "C" __attribute__((visibility("default")))

// the launch of mfn_split_pack with one one-thread block: the grid-stride loop covers every item
EMU_API void emu_split_pack(const float* src, long long src_bs, int N, int C, int H, int W, unsigned char* dst,
                            int dst_channels, int dst_c0) {
  blockDim = dim3(1);
  threadIdx = dim3(0);
  gridDim = dim3(1);
  blockIdx = dim3(0);
  split_pack_kernel(src, src_bs, C, dst, sa::groups(dst_channels), dst_c0 / 8, N, (long long)H * W);
}
