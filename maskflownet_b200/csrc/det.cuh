// det.cuh -- arithmetic of the deterministic backward mode (det_bwd.cu, the *_det entry points of maskflow_b200.h): 64-bit
// fixed-point accumulation for the scatter-shaped gradients.  Device functions only and no CUDA runtime header, so that the
// host emulation (tests/host_emu/det_emu.cpp) compiles the same arithmetic.
//
// A scatter adds fp32 contributions c, |c| <= B, into destinations that each receive at most `fanin` of them.  Every c is
// rounded to a multiple of 2^-s and added as a two's-complement int64 with an integer atomic; integer addition is
// associative, so the sum does not depend on the order in which threads run.  One pass converts the sums back to fp32.
//
// Scale.  B < 2^e (frexp) and fanin < 2^k (k = fanin bit length, computed on the host from the shape), s = 61 - k - e,
// capped at 126 so that 2^s is an fp32 power of two.  Then |c 2^s| < 2^(61-k) and a destination's sum stays below
// fanin (2^(61-k) + 1/2) < 2^62: no sum can overflow, even when every source lands on one element.  The factor-2 headroom
// below 2^63 absorbs the fp32 rounding of B and of the contributions themselves.
//
// Error.  Rounding one contribution costs at most 2^-(s+1) = 2^(k+e-62) <= 4 fanin B 2^-62, so an element that receives n
// contributions differs from the exact (float64) sum of its fp32 contributions by at most
//     n 2^(k+e-62)  (<= fanin^2 B 2^-60)     plus half an fp32 ulp of the result (the final conversion),
// e.g. 36 contributions at B = 1 with fanin = 4*448*1024 (k = 21): 36 * 2^-40 ~ 3e-11 absolute.  With s capped at 126
// (B < 2^(-65-k)) the bound is n 2^-127.
//
// A bound that is NaN, inf or beyond the fp32 range marks the scale as non-finite: the scatter adds nothing and the
// conversion writes NaN to every element, so NaN / inf gradients show up as NaN instead of wrapped integers.
#pragma once

#ifdef MFN_HOST_EMULATION
// host stand-ins of the device intrinsics used below; with one thread at a time the atomic is a plain add
#include <cmath>
#include <cstring>
template <typename To, typename From>
static inline To det_bit_cast_(From v) {
  To r;
  std::memcpy(&r, &v, sizeof r);
  return r;
}
static inline unsigned __float_as_uint(float f) { return det_bit_cast_<unsigned>(f); }
static inline float __uint_as_float(unsigned u) { return det_bit_cast_<float>(u); }
static inline float __int_as_float(int i) { return det_bit_cast_<float>(i); }
static inline double __longlong_as_double(long long i) { return det_bit_cast_<double>(i); }
static inline long long __float2ll_rn(float v) { return std::llrint(v); }   // round to nearest even, like the device
static inline unsigned long long atomicAdd(unsigned long long* p, unsigned long long v) {
  const unsigned long long old = *p;
  *p = old + v;
  return old;
}
#endif

namespace mfn {

constexpr int kDetHeaderBytes = 256;   // start of every det workspace: the bound words (unsigned[0..1]), then padding
constexpr int kDetSlices = 64;         // slices per plane of the deterministic preprocess plane sums (independent of the GPU)

struct FixedScale {
  float up;       // 2^s
  double down;    // 2^-s
  bool finite;
};

// |v| as the bit pattern of a non-negative float: orders like the value, with +inf above every finite value and every NaN
// above +inf, so an unsigned max over it is a max that keeps NaN.
__device__ __forceinline__ unsigned det_abs_bits(float v) { return __float_as_uint(v) & 0x7fffffffu; }

// the finite scale 2^s for an exponent known in advance (-126 <= s <= 126), e.g. from a static bound on the contributions
__device__ __forceinline__ FixedScale det_fixed_scale(int s) {
  FixedScale f;
  f.up = __int_as_float((s + 127) << 23);
  f.down = __longlong_as_double((long long)(1023 - s) << 52);
  f.finite = true;
  return f;
}

// nb = 1: B = bound[0]; nb = 2: B = bound[0] * bound[1] (in double, so that the product itself cannot overflow)
__device__ __forceinline__ FixedScale det_scale(const unsigned* __restrict__ bound, int nb, int fanin_bits) {
  double b = (double)__uint_as_float(bound[0]);
  if (nb == 2) b *= (double)__uint_as_float(bound[1]);
  const bool finite = b <= 3.4028234663852886e38;   // FLT_MAX; false for NaN and inf
  int e = 0;
  if (finite && b > 0.0) frexp(b, &e);
  int s = 61 - fanin_bits - e;
  if (s > 126) s = 126;                    // s >= 61 - 40 - 128 for every shape the entry points accept
  FixedScale f = det_fixed_scale(s);
  f.finite = finite;
  return f;
}

__device__ __forceinline__ unsigned long long det_to_fixed(float c, const FixedScale& f) {
  return (unsigned long long)__float2ll_rn(c * f.up);
}

__device__ __forceinline__ float det_from_fixed(unsigned long long acc, const FixedScale& f) {
  return f.finite ? (float)((double)(long long)acc * f.down) : __int_as_float(0x7fc00000);
}

// fixed-point scatter of one contribution (no-op for a non-finite scale: the conversion writes NaN anyway)
__device__ __forceinline__ void det_scatter(unsigned long long* p, float c, const FixedScale& f) {
  if (f.finite) atomicAdd(p, det_to_fixed(c, f));
}

// bit length of n: n < 2^k
static inline int det_bits(long long n) {
  int k = 0;
  while (k < 62 && (1LL << k) <= n) ++k;
  return k;
}

}  // namespace mfn
