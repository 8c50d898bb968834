// denoise_emu.cpp -- TEST INFRASTRUCTURE ONLY.  Compiles video denoising (maskflownet_b200/csrc/denoise.cu) for the host
// through cuda_shim.h and runs the launches of mfn_denoise_frames and mfn_noise_sigma one thread at a time.  Each CTA's
// phases (chain start, chain step, accumulation, store) run over its threads in turn, in the kernel's order, with the
// per-thread sums kept here; C ABI for tests/test_denoise.py.
//   g++ -O1 -ffp-contract=off -shared -fPIC -I tests/host_emu denoise_emu.cpp
#define MFN_HOST_EMULATION 1
#include <cstring>
#include <vector>

#include "cuda_shim.h"

// the vector type and the bit cast the kernels use; floorf, rintf, expf, fminf and fmaxf are the C library's
struct float2 {
  float x, y;
};
static inline float __int_as_float(int v) {
  float f;
  std::memcpy(&f, &v, 4);
  return f;
}

#include "../../maskflownet_b200/csrc/denoise.cu"

using namespace mfn;

#define EMU_API extern "C" __attribute__((visibility("default")))

EMU_API void emu_denoise_frames(const unsigned char* frames, const float* flow_fw, const float* flow_bw,
                                unsigned char* out, int S, int H, int W, int t0, int N, int t_lo, int t_hi, int radius,
                                int patch, float sigma, float h_factor, float alpha, float beta) {
  DnArgs a;
  a.frames = frames;
  a.fw = reinterpret_cast<const float2*>(flow_fw);
  a.bw = reinterpret_cast<const float2*>(flow_bw);
  a.out = out;
  a.S = S, a.H = H, a.W = W, a.t0 = t0, a.t_lo = t_lo, a.t_hi = t_hi, a.R = radius, a.r = patch;
  a.alpha = alpha, a.beta = beta;
  a.two_s2 = 2.f * (sigma * sigma);
  const float hs = h_factor * sigma;
  a.h2 = hs * hs;
  const int tiles_x = (W + kDnTile - 1) / kDnTile, tiles_y = (H + kDnTile - 1) / kDnTile;
  std::vector<float> sm(8 * (size_t)dn_halo(patch) * dn_halo(patch));
  const DnShared s = dn_shared(sm.data(), patch);
  static float acc[kDnThreads][4];
  for (int n = 0; n < N; ++n) {
    const int t = t0 + n;
    for (int b = 0; b < tiles_x * tiles_y; ++b) {
      const int bx0 = (b % tiles_x) * kDnTile, by0 = (b / tiles_x) * kDnTile;
      for (int i = 0; i < kDnThreads; ++i) acc[i][0] = acc[i][1] = acc[i][2] = acc[i][3] = 0.f;
      for (int dir = 0; dir < 2; ++dir) {
        const bool fwd = dir == 0;
        const int K = dn_steps(a, t, fwd);
        if (K <= 0) continue;
        for (int i = 0; i < s.P; ++i) dn_start(a, t, bx0, by0, i, s);
        for (int k = 1; k <= K; ++k) {
          for (int i = 0; i < s.P; ++i) dn_step(a, t, k, fwd, i, s);
          for (int ty = 0; ty < kDnTile; ++ty)
            for (int tx = 0; tx < kDnTile; ++tx)
              if (bx0 + tx < W && by0 + ty < H) dn_accumulate(a, tx, ty, s, acc[ty * kDnTile + tx]);
        }
      }
      for (int ty = 0; ty < kDnTile; ++ty)
        for (int tx = 0; tx < kDnTile; ++tx)
          if (bx0 + tx < W && by0 + ty < H) dn_store(a, t, n, bx0 + tx, by0 + ty, acc[ty * kDnTile + tx]);
    }
  }
}

// mfn_noise_sigma's launch: per frame the 1024 threads' sums, the tree, the float64 expression; sums (F) the exact S
EMU_API void emu_noise_sigma(const unsigned char* frames, double* sigma, long long* sums, int F, int H, int W) {
  static long long sh[kNoiseThreads];
  for (int f = 0; f < F; ++f) {
    const unsigned char* fr = frames + (size_t)f * 3 * H * W;
    for (int t = 0; t < kNoiseThreads; ++t) sh[t] = noise_thread_sum(fr, H, W, t, kNoiseThreads);
    for (int stride = kNoiseThreads / 2; stride > 0; stride >>= 1)
      for (int t = 0; t < kNoiseThreads; ++t) noise_tree_step(sh, t, stride);
    sums[f] = sh[0];
    sigma[f] = noise_sigma_of(sh[0], H, W);
  }
}
