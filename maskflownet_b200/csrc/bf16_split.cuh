// bf16_split.cuh -- the bf16 hi/lo split every tensor-core contraction rests on (DESIGN section 4), on its own so that the
// element-wise kernels that store split operands (split_act.cu) also build for the host: under MFN_HOST_EMULATION the
// one instruction, cvt.rn.bf16x2.f32, is the host stand-in cvt_bf16x2_rn(first, second) that
// tests/host_emu/split_act_emu.cpp supplies.  ptx.cuh includes it: one definition for every kernel.
#pragma once
#include <stdint.h>

namespace mfn {

// (a, b) fp32 -> packed bf16x2 "hi" (a in the low half: the lower k index of an MMA fragment register) and the bf16x2 of
// the remainders "lo", both rounded to nearest even.  Every contraction sums hi*hi + hi*lo + lo*hi in fp32.
__device__ __forceinline__ void split_pair(float a, float b, uint32_t& hi, uint32_t& lo) {
#ifndef MFN_HOST_EMULATION
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(hi) : "f"(b), "f"(a));
#else
  hi = cvt_bf16x2_rn(a, b);
#endif
  const float ah = __uint_as_float(hi << 16), bh = __uint_as_float(hi & 0xffff0000u);
#ifndef MFN_HOST_EMULATION
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(lo) : "f"(b - bh), "f"(a - ah));
#else
  lo = cvt_bf16x2_rn(a - ah, b - bh);
#endif
}

// (a, b) fp32 -> packed bf16x2 rounded to nearest even: the "hi" of split_pair alone, the operand of the bf16 mode
__device__ __forceinline__ uint32_t bf16_pair(float a, float b) {
  uint32_t r;
#ifndef MFN_HOST_EMULATION
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(b), "f"(a));
#else
  r = cvt_bf16x2_rn(a, b);
#endif
  return r;
}

}  // namespace mfn
