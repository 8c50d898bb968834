// interp_emu.cpp -- TEST INFRASTRUCTURE ONLY.  Compiles frame interpolation (maskflownet_b200/csrc/interp.cu) for the host
// through cuda_shim.h and runs mfn_interpolate_frames' launch sequence (zeroed accumulators, splat, normalise per time step)
// one thread at a time, the splat's threads in a caller-chosen order; C ABI for tests/test_interpolate.py.
//   g++ -O1 -ffp-contract=off -shared -fPIC -I tests/host_emu interp_emu.cpp
#define MFN_HOST_EMULATION 1
#include <vector>

#include "cuda_shim.h"

// the vector types the kernels read; fmaf, floorf and rintf are the C library's
struct float2 {
  float x, y;
};
struct ulonglong2 {
  unsigned long long x, y;
};

#include "../../maskflownet_b200/csrc/interp.cu"

using namespace mfn;

#define EMU_API extern "C" __attribute__((visibility("default")))

EMU_API int emu_interp_weight_shift(int H, int W) { return interp_weight_shift(H, W); }

// order: null (ascending), or a permutation of the splat's 2 * N * ceil(HW / 256) * 256 threads, numbered
// ((z * N + n) * blocks + block) * 256 + thread.  acc_out (N,H,W,4), optional: the last time step's accumulators.
EMU_API void emu_interpolate_frames(const unsigned char* img0, const unsigned char* img1, const float* flow_fw,
                                    const float* flow_bw, const unsigned char* occ_fw, const unsigned char* occ_bw,
                                    unsigned char* out, int N, int H, int W, const float* times, int T, float occ_weight,
                                    const long long* order, long long* acc_out) {
  const int HW = H * W;
  const unsigned blocks = (HW + 255) / 256;
  const long long threads = 2LL * N * blocks * 256;
  const int s_w = interp_weight_shift(H, W);
  std::vector<unsigned long long> acc(4LL * N * HW);
  for (int k = 0; k < T; ++k) {
    std::fill(acc.begin(), acc.end(), 0ull);
    blockDim = dim3(256);
    gridDim = dim3(blocks, N, 2);
    for (long long j = 0; j < threads; ++j) {
      const long long g = order ? order[j] : j;
      const long long b = g / 256;
      threadIdx = dim3((unsigned)(g % 256));
      blockIdx = dim3((unsigned)(b % blocks), (unsigned)((b / blocks) % N), (unsigned)(b / blocks / N));
      splat_kernel(img0, img1, reinterpret_cast<const float2*>(flow_fw), reinterpret_cast<const float2*>(flow_bw), occ_fw,
                   occ_bw, acc.data(), H, W, times[k], occ_weight, s_w);
    }
    gridDim = dim3(blocks, N);
    for (unsigned n = 0; n < (unsigned)N; ++n)
      for (unsigned b = 0; b < blocks; ++b)
        for (unsigned t = 0; t < 256; ++t) {
          blockIdx = dim3(b, n);
          threadIdx = dim3(t);
          normalise_kernel(acc.data(), img0, img1, out, H, W, T, k, times[k], s_w);
        }
  }
  if (acc_out) std::copy(acc.begin(), acc.end(), reinterpret_cast<unsigned long long*>(acc_out));
}
