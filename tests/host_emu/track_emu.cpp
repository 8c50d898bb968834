// track_emu.cpp -- TEST INFRASTRUCTURE ONLY.  Compiles dense point tracking (maskflownet_b200/csrc/track.cu) for the host
// through cuda_shim.h and runs the launches of mfn_track_texture, mfn_track_advance and mfn_track_seed one thread at a
// time.  The seed kernel's phases run over its 1024 threads in turn, with the block scans done here in between;
// C ABI for tests/test_tracking.py.
//   g++ -O1 -ffp-contract=off -shared -fPIC -I tests/host_emu track_emu.cpp
#define MFN_HOST_EMULATION 1
#include <cstring>
#include <vector>

#include "cuda_shim.h"

// the vector type and the bit casts the kernels use; floorf, rintf and sqrt are the C library's
struct float2 {
  float x, y;
};
static inline float __int_as_float(int v) {
  float f;
  std::memcpy(&f, &v, 4);
  return f;
}
static inline long long __double_as_longlong(double v) {
  long long r;
  std::memcpy(&r, &v, 8);
  return r;
}
static inline unsigned long long atomicMax(unsigned long long* p, unsigned long long v) {
  const unsigned long long old = *p;
  if (v > old) *p = v;
  return old;
}

#include "../../maskflownet_b200/csrc/track.cu"

using namespace mfn;

#define EMU_API extern "C" __attribute__((visibility("default")))

EMU_API void emu_track_texture(const unsigned char* frames, double* lambda2, double* lambda_max, int F, int H, int W,
                               int h) {
  const int Gx = W / h, G = Gx * (H / h);
  std::memset(lambda_max, 0, sizeof(double) * F);
  if (G == 0) return;
  blockDim = dim3(256);
  gridDim = dim3((G + 255) / 256, F);
  for (unsigned f = 0; f < gridDim.y; ++f)
    for (unsigned b = 0; b < gridDim.x; ++b)
      for (unsigned t = 0; t < 256; ++t) {
        blockIdx = dim3(b, f);
        threadIdx = dim3(t);
        track_texture_kernel(frames, lambda2, reinterpret_cast<unsigned long long*>(lambda_max), H, W, h, Gx, G);
      }
}

EMU_API void emu_track_advance(const float* flow_fw, const float* flow_bw, float* pos, unsigned char* status,
                               unsigned char* cells, int K, int H, int W, int h, float alpha, float beta, float alpha_b,
                               float beta_b) {
  const int Gx = W / h, Gy = H / h;
  std::memset(cells, 0, (size_t)Gx * Gy);
  blockDim = dim3(256);
  gridDim = dim3((K + 255) / 256);
  for (unsigned b = 0; b < gridDim.x; ++b)
    for (unsigned t = 0; t < 256; ++t) {
      blockIdx = dim3(b);
      threadIdx = dim3(t);
      track_advance_kernel(reinterpret_cast<const float2*>(flow_fw), reinterpret_cast<const float2*>(flow_bw),
                           reinterpret_cast<float2*>(pos), status, cells, K, H, W, h, Gx, Gy, alpha, beta, alpha_b,
                           beta_b);
    }
}

// track_seed_kernel's phases over T = 1024 threads; the exclusive scans of the per-thread counts are done here.
EMU_API void emu_track_seed(const double* lambda2, const double* lambda_max, const float* queries, int M, float* pos,
                            unsigned char* status, unsigned char* cells, int* frame, int* dropped, int K, int H, int W,
                            int h, float tau) {
  const int T = kTrackSeedThreads, Gx = W / h, Gy = H / h, G = Gx * Gy;
  const int f = *frame;
  float2* p2 = reinterpret_cast<float2*>(pos);
  std::vector<int> freelist(K), c0(T), f0(T);
  for (int t = 0; t < T; ++t) track_seed_births(t, T, queries, M, f, p2, status, cells, H, W, h, Gx, Gy);
  const double thr = (double)tau * *lambda_max;
  int C = 0, Fr = 0;
  for (int t = 0; t < T; ++t) {
    c0[t] = C;
    C += track_count_candidates(t, T, lambda2, cells, G, thr);
    f0[t] = Fr;
    Fr += track_count_free(t, T, status, M, K);
  }
  for (int t = 0; t < T; ++t) track_write_freelist(t, T, status, M, K, f0[t], C, freelist.data());
  for (int t = 0; t < T; ++t) track_assign(t, T, lambda2, cells, G, thr, c0[t], Fr, freelist.data(), p2, status, h, Gx);
  *dropped = C > Fr ? C - Fr : 0;
  *frame = f + 1;
}
