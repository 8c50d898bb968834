// common.cuh -- shared host/device helpers for libmaskflow_b200 (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/maskflow_b200.h"
#include "device_caps.h"
#include "sampling.cuh"

namespace mfn {

// ---- host-side error / bookkeeping (defined in api.cu) ------------------------------------------------
int fail(int code, const char* fmt, ...);
int check_launch(const char* kernel_name);  // cudaGetLastError -> return code, bumps launch counter
void note_kernel(const char* name);

// process-wide tuning / test knobs (mfn_set_tuning)
struct Tuning {
  int corr_grid_cap = 0;      // > 0: cap the persistent grid of the MMA correlation kernels (tests force long tile runs)
  int corr_disable_ring = 0;  // 1: use the tile kernel even for C <= 32
  int conv_wgmma = 1;          // 1: 3x3 convolutions run on wgmma (conv3x3_wgmma.cu), 0: mma.sync kernel
  int conv_grid_cap = 0;      // persistent wgmma convolution: CTAs (0 = one per SM); tests force long per-CTA tile runs
  int conv_wgmma_min_w = 1;    // narrower images stay on the mma.sync kernel (a 128-pixel M tile would be mostly padding)
  int corr_ring_th = 8;       // tile height of the strip-marching kernel: 4 (8 warps, 2 CTAs/SM) or 8 (16 warps, 1 CTA/SM)
  int corr_rb = 1;            // 1: C > 32 correlations run on the row-block kernel (corr_rb.cu); 2: also C <= 32 when the TMA kernel declines; 0: chunked tile kernel
  int warp_lin_fch = 0;       // > 0: channels per thread of warp_lin_kernel (a multiple of 8; default: 16 / 32 / 64 by level size)
  int conv_as = 0;            // 2: wide wgmma layers keep 2 input stages (more weight stages); default 3
  int conv_splitk = 1;        // 0: never split K; 1: plan decides (<= 8 parts); k > 1: cap on the number of parts
  int corr_rb_twb = 0;        // 2: force 16-pixel strips in the row-block kernel (two CTAs per SM when the tile fits 113 KB)
  int corr_rb_rows = 0;       // > 0: start the row-block kernel's RB search at this value (4 / 2 / 1)
  int corr_tma = 1;           // 1: C <= 32 correlations run on the TMA pipeline kernel (corr_tma.cu) when the shape fits
  int warp_lin = 1;           // 1: mfn_warp_mask_forward_resample evaluates every pixel through linearity (warp_lin.cu); 0: border list
  int corr_ts_lo = 0, corr_ts_hi = 0;   // development: device pointer (two halves) of the timeline buffer of corr_tma_kernel, 0 = off
  int corr_dbg = 0;           // profiling aid for the ring kernel: 2 = producers idle, 4 = no epilogue, 8 = no MMA (results invalid)
};
Tuning& tuning();

static inline cudaStream_t as_stream(void* s) { return reinterpret_cast<cudaStream_t>(s); }

#define MFN_REQUIRE(cond, code, ...)                   \
  do {                                                 \
    if (!(cond)) return ::mfn::fail(code, __VA_ARGS__); \
  } while (0)

static inline bool aligned(const void* p, size_t a) { return (reinterpret_cast<uintptr_t>(p) % a) == 0; }

// blocks of a grid-stride element-wise launch: enough for `total` items, at most 16 per SM
static inline unsigned grid_for(long long total, int threads) {
  long long b = (total + threads - 1) / threads;
  const long long cap = (long long)kNumSMs * 16;
  return (unsigned)(b < cap ? (b > 0 ? b : 1) : cap);
}


// cudaFuncAttributeMaxDynamicSharedMemorySize is per function AND per device (a process may drive several GPUs: ops._call
// switches the device per tensor): remember the largest opt-in per device, re-issue it when a launch needs more.
struct SmemOptIn {
  int bytes[64] = {};
};
template <typename K>
static inline cudaError_t ensure_dyn_smem(K kernel, int bytes, SmemOptIn& st) {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) dev = -1;
  if (dev >= 0 && dev < 64 && st.bytes[dev] >= bytes) return cudaSuccess;
  const cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
  if (e == cudaSuccess && dev >= 0 && dev < 64) st.bytes[dev] = bytes;
  return e;
}

// warp_lin.cu: K3 through linearity, exact for both border rules; -1 = the extended wgmma convolution does not fit
long long warp_lin_workspace_bytes(int N, int F, int H, int W);
int launch_warp_lin(const float* x, const float* flow_c, const float* mask_c, const float* weight, const void* packed_weight,
                    const float* bias, const float* tradeoff, void* workspace, float* out, float* fup, float* mup, int N,
                    int C, int H, int W, int F, int up, float fs, float ls, float slope, int border_mode, cudaStream_t st);

// corr_rb.cu: returns -1 when no configuration fits shared memory
int launch_corr_rb(int md, const float* d1, const float* d2, float* out, int N, int C, int H, int W, long long obs,
                   float slope, cudaStream_t st);

// corr_tma.cu: returns -1 when the shape / alignment does not fit (caller falls back to the LDG kernels)
int launch_corr_tma(int md, const float* d1, const float* d2, float* out, int N, int C, int H, int W, long long obs,
                    float slope, cudaStream_t st);

// det_bwd.cu: the shared passes of the deterministic backward mode (arithmetic in det.cuh)
int det_launch_abs_max(const float* v, long long n, unsigned* bound, cudaStream_t st);
int det_launch_pixel_abs_sum_max(const float* g, int N, int F, long long HW, unsigned* bound, cudaStream_t st);
int det_launch_fixed_to_float(const unsigned long long* acc, float* out, long long n, const unsigned* bound, int nb,
                              int fanin_bits, cudaStream_t st);
int det_launch_ordered_sum(const float* part, int nparts, long long part_stride, long long elem_stride, float* out,
                           long long n, int accumulate, cudaStream_t st);
int det_check_workspace(const char* fn, const void* ws, long long bytes, long long need);

// ---- device helpers ---------------------------------------------------------------------------------
__device__ __forceinline__ float leaky(float v, float slope) { return v > 0.f ? v : v * slope; }

// sigmoidf_, upsample_taps / upsample_at and the BilinearSampler taps: sampling.cuh (shared with the host emulation)

// Bilinear tap of the deformable convolution: weights + indices for one real position (h, w).
// valid == false means the tap contributes zero (see MFN_BORDER_* in maskflow_b200.h).
struct Tap {
  int h0, h1, w0, w1;
  float lh, lw;  // fractional parts (already zeroed in the collapsed regime)
  bool valid;
  bool c00, c01, c10, c11;  // per-corner validity (always true in MXNET15 mode when valid)
};

template <int BORDER>
__device__ __forceinline__ Tap make_tap(float h, float w, int H, int W) {
  Tap t;
  if (BORDER == MFN_BORDER_MXNET15) {
    t.valid = (h >= 0.f) && (w >= 0.f) && (h < (float)H) && (w < (float)W);
    int h0 = (int)floorf(h), w0 = (int)floorf(w);
    if (h0 >= H - 1) {
      h0 = H - 1;
      t.h1 = h0;
      t.lh = 0.f;
    } else {
      t.h1 = h0 + 1;
      t.lh = h - (float)h0;
    }
    if (w0 >= W - 1) {
      w0 = W - 1;
      t.w1 = w0;
      t.lw = 0.f;
    } else {
      t.w1 = w0 + 1;
      t.lw = w - (float)w0;
    }
    t.h0 = h0;
    t.w0 = w0;
    if (!t.valid) {  // keep indices in range so that speculative loads stay legal
      t.h0 = t.h1 = t.w0 = t.w1 = 0;
      t.lh = t.lw = 0.f;
    }
    t.c00 = t.c01 = t.c10 = t.c11 = t.valid;
  } else {
    t.valid = (h > -1.f) && (w > -1.f) && (h < (float)H) && (w < (float)W);
    const int h0 = (int)floorf(h), w0 = (int)floorf(w);
    t.lh = h - (float)h0;
    t.lw = w - (float)w0;
    const bool hin0 = h0 >= 0, hin1 = h0 + 1 <= H - 1, win0 = w0 >= 0, win1 = w0 + 1 <= W - 1;
    t.c00 = t.valid && hin0 && win0;
    t.c01 = t.valid && hin0 && win1;
    t.c10 = t.valid && hin1 && win0;
    t.c11 = t.valid && hin1 && win1;
    t.h0 = max(min(h0, H - 1), 0);
    t.h1 = max(min(h0 + 1, H - 1), 0);
    t.w0 = max(min(w0, W - 1), 0);
    t.w1 = max(min(w0 + 1, W - 1), 0);
    if (!t.valid) t.lh = t.lw = 0.f;
  }
  return t;
}

__device__ __forceinline__ float tap_sample(const Tap& t, const float* __restrict__ plane, int W) {
  const float hh = 1.f - t.lh, hw = 1.f - t.lw;
  float v = 0.f;
  if (t.c00) v += hh * hw * __ldg(plane + (size_t)t.h0 * W + t.w0);
  if (t.c01) v += hh * t.lw * __ldg(plane + (size_t)t.h0 * W + t.w1);
  if (t.c10) v += t.lh * hw * __ldg(plane + (size_t)t.h1 * W + t.w0);
  if (t.c11) v += t.lh * t.lw * __ldg(plane + (size_t)t.h1 * W + t.w1);
  return v;
}

}  // namespace mfn
