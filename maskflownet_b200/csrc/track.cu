// track.cu -- dense point tracking through a video (Sundaram, Brox and Keutzer, ECCV 2010): tracks chained along the
// forward flow, stopped by the forward-backward check (occlusion) or by the flow's gradient (motion boundary), and
// reseeded on a grid wherever a textured cell is left uncovered.
//
//   mfn_track_texture   frames (F,H,W,3) uint8  ->  lambda2 (F,Gy,Gx), lambda_max (F) float64
//     cudaMemsetAsync of lambda_max;  track_texture_kernel, grid (cells / 256, F): one thread per seed point, the smaller
//     eigenvalue of its 5x5 structure tensor (integers, then float64), the frame's max by atomicMax on the float64 bits
//     (non-negative doubles order like their bits, so the max does not depend on the order of the atomics).
//   mfn_track_advance   flow_fw, flow_bw (H,W,2) of frames k -> k+1, slot state of frame k  ->  state of frame k+1, cells
//     cudaMemsetAsync of the cell occupancy;  track_advance_kernel, grid (K / 256): one thread per slot.
//   mfn_track_seed      lambda2, lambda_max of the frame, queries, state  ->  the frame's births, dropped count, frame + 1
//     track_seed_kernel, one CTA of 1024 threads: query births, then one block scan over the candidate cells and one over
//     the free slots, so the n-th candidate in row-major cell order takes the n-th free slot.
// The rule is in include/maskflow_b200.h.  Integer bookkeeping only, no float atomics: the result is deterministic.  No
// allocation and no host synchronisation, and the frame index lives in device memory, so a sequence of steps is
// capture-safe and a graph replay equals the eager chain.
//
// The file also builds for the host (MFN_HOST_EMULATION: tests/host_emu/track_emu.cpp), one thread at a time.  The seed
// kernel's phases are separate functions, so the host runs them with its own scan in between.
#ifdef MFN_HOST_EMULATION
#include "cuda_shim.h"
#else
#include <math.h>

#include "common.cuh"
#endif
#include "flowcheck.cuh"   // fb_sample, fb_consistent

namespace mfn {

enum : unsigned char {
  kTrackEmpty = 0,      // no track in this slot in this frame
  kTrackTracked = 1,    // a track continued into this frame
  kTrackBorn = 2,       // a track started in this frame (seed or query)
  kTrackLeft = 3,       // the track's last frame was the previous one: its target was non-finite or left the frame
  kTrackOccluded = 4,   // ... ended by the forward-backward check
  kTrackBoundary = 5,   // ... ended by the motion-boundary test
};
constexpr int kTrackSeedThreads = 1024;

__device__ __forceinline__ bool track_alive(unsigned char s) { return s == kTrackTracked || s == kTrackBorn; }

// ---- texture ------------------------------------------------------------------------------------------------------
__device__ __forceinline__ int track_grey(const unsigned char* __restrict__ f, int W, int x, int y) {
  const unsigned char* p = f + 3 * ((size_t)y * W + x);
  return (int)__ldg(p) + (int)__ldg(p + 1) + (int)__ldg(p + 2);
}

// lambda_2 of the structure tensor summed over the 5x5 window (clamped) around (sx, sy): the gradients and sums are exact
// int32 (|g| <= 765, 25 g^2 < 2^24), and every float64 intermediate is an integer or half-integer below 2^53, so the
// result is the correctly rounded value of one subtraction and one square root: bit-identical to numpy.
__device__ __forceinline__ double track_lambda2(const unsigned char* __restrict__ f, int H, int W, int sx, int sy) {
  int a = 0, b = 0, c = 0;
  for (int dy = -2; dy <= 2; ++dy) {
    const int y = min(max(sy + dy, 0), H - 1);
    const int ym = max(y - 1, 0), yp = min(y + 1, H - 1);
    for (int dx = -2; dx <= 2; ++dx) {
      const int x = min(max(sx + dx, 0), W - 1);
      const int gx = track_grey(f, W, min(x + 1, W - 1), y) - track_grey(f, W, max(x - 1, 0), y);
      const int gy = track_grey(f, W, x, yp) - track_grey(f, W, x, ym);
      a += gx * gx;
      b += gx * gy;
      c += gy * gy;
    }
  }
  const double h = 0.5 * ((double)a - (double)c);
  const double l2 = 0.5 * ((double)a + (double)c) - sqrt(h * h + (double)b * (double)b);
  return l2 > 0.0 ? l2 : 0.0;
}

// grid (ceil(G / blockDim), F): lambda2[f, c] for the seed point of cell c = j Gx + i, ((i h + h/2), (j h + h/2))
__global__ void __launch_bounds__(256)
    track_texture_kernel(const unsigned char* __restrict__ frames, double* __restrict__ lambda2,
                         unsigned long long* __restrict__ lambda_max, int H, int W, int h, int Gx, int G) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= G) return;
  const size_t f = blockIdx.y;
  const int j = c / Gx, i = c - j * Gx;
  const double l2 = track_lambda2(frames + f * 3 * (size_t)H * W, H, W, i * h + h / 2, j * h + h / 2);
  lambda2[f * G + c] = l2;
  atomicMax(lambda_max + f, (unsigned long long)__double_as_longlong(l2));
}

// ---- advance ------------------------------------------------------------------------------------------------------
// The status of a track at p (inside the frame) in the next frame, and its position q there when it is TRACKED.
__device__ __forceinline__ unsigned char track_rule(const float2* __restrict__ flow_fw, const float2* __restrict__ flow_bw,
                                                    int H, int W, float2 p, float alpha, float beta, float alpha_b,
                                                    float beta_b, float2* q) {
  const float2 w = fb_sample(flow_fw, H, W, p.x, p.y);
  const float qx = p.x + w.x, qy = p.y + w.y;
  if (!(qx >= 0.f && qx <= (float)(W - 1) && qy >= 0.f && qy <= (float)(H - 1))) return kTrackLeft;
  if (!fb_consistent(w, fb_sample(flow_bw, H, W, qx, qy), alpha, beta)) return kTrackOccluded;
  // motion boundary: central differences of flow_fw at the pixel nearest p, neighbours clamped to the frame
  const int cx = min(max((int)rintf(p.x), 0), W - 1), cy = min(max((int)rintf(p.y), 0), H - 1);
  const int xl = max(cx - 1, 0), xr = min(cx + 1, W - 1), yl = max(cy - 1, 0), yr = min(cy + 1, H - 1);
  float2 gx = float2{0.f, 0.f}, gy = float2{0.f, 0.f};
  if (xr > xl) {
    const float2 l = __ldg(flow_fw + (size_t)cy * W + xl), r = __ldg(flow_fw + (size_t)cy * W + xr);
    const float d = (float)(xr - xl);
    gx = float2{(r.x - l.x) / d, (r.y - l.y) / d};
  }
  if (yr > yl) {
    const float2 u = __ldg(flow_fw + (size_t)yl * W + cx), v = __ldg(flow_fw + (size_t)yr * W + cx);
    const float d = (float)(yr - yl);
    gy = float2{(v.x - u.x) / d, (v.y - u.y) / d};
  }
  const float g = gx.x * gx.x + gx.y * gx.y + gy.x * gy.x + gy.y * gy.y;
  if (!(g <= alpha_b * (w.x * w.x + w.y * w.y) + beta_b)) return kTrackBoundary;
  *q = float2{qx, qy};
  return kTrackTracked;
}

// grid (ceil(K / blockDim)): slot s in frame k -> k+1.  A live slot takes track_rule's status (NaN position unless
// TRACKED) and a TRACKED one marks its cell; every other slot becomes EMPTY.
__global__ void __launch_bounds__(256)
    track_advance_kernel(const float2* __restrict__ flow_fw, const float2* __restrict__ flow_bw, float2* __restrict__ pos,
                         unsigned char* __restrict__ status, unsigned char* __restrict__ cells, int K, int H, int W, int h,
                         int Gx, int Gy, float alpha, float beta, float alpha_b, float beta_b) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= K) return;
  const float nan = __int_as_float(0x7fc00000);
  float2 q = float2{nan, nan};
  unsigned char next = kTrackEmpty;
  if (track_alive(status[s])) next = track_rule(flow_fw, flow_bw, H, W, pos[s], alpha, beta, alpha_b, beta_b, &q);
  if (next == kTrackTracked) {
    const int i = (int)floorf(q.x) / h, j = (int)floorf(q.y) / h;
    if (i < Gx && j < Gy) cells[(size_t)j * Gx + i] = 1;
  }
  pos[s] = q;
  status[s] = next;
}

// ---- seed: the phases of track_seed_kernel, thread t of T ----------------------------------------------------------
// Query i (row (t, x, y) of `queries`) is born in frame f == t: BORN at (x, y) inside [0,W-1] x [0,H-1] (its cell is then
// covered), LEFT with a NaN position otherwise.
__device__ __forceinline__ void track_seed_births(int t, int T, const float* __restrict__ queries, int M, int f,
                                                  float2* __restrict__ pos, unsigned char* __restrict__ status,
                                                  unsigned char* __restrict__ cells, int H, int W, int h, int Gx, int Gy) {
  for (int k = t; k < M; k += T) {
    if (!(queries[3 * k] == (float)f)) continue;
    const float x = queries[3 * k + 1], y = queries[3 * k + 2];
    if (x >= 0.f && x <= (float)(W - 1) && y >= 0.f && y <= (float)(H - 1)) {
      pos[k] = float2{x, y};
      status[k] = kTrackBorn;
      const int i = (int)floorf(x) / h, j = (int)floorf(y) / h;
      if (i < Gx && j < Gy) cells[(size_t)j * Gx + i] = 1;
    } else {
      const float nan = __int_as_float(0x7fc00000);
      pos[k] = float2{nan, nan};
      status[k] = kTrackLeft;
    }
  }
}

// thread t's contiguous share [b, e) of n items, in order
__device__ __forceinline__ void track_range(int t, int T, int n, int* b, int* e) {
  const int chunk = (n + T - 1) / T;
  *b = min(t * chunk, n);
  *e = min(*b + chunk, n);
}

__device__ __forceinline__ bool track_candidate(const double* __restrict__ lambda2, const unsigned char* __restrict__ cells,
                                                int c, double thr) {
  const double l = lambda2[c];
  return !cells[c] && l > 0.0 && l >= thr;
}

__device__ __forceinline__ int track_count_candidates(int t, int T, const double* __restrict__ lambda2,
                                                      const unsigned char* __restrict__ cells, int G, double thr) {
  int b, e, n = 0;
  track_range(t, T, G, &b, &e);
  for (int c = b; c < e; ++c) n += track_candidate(lambda2, cells, c, thr);
  return n;
}

// the free slots are the dense slots M..K-1 that are EMPTY after the advance
__device__ __forceinline__ int track_count_free(int t, int T, const unsigned char* __restrict__ status, int M, int K) {
  int b, e, n = 0;
  track_range(t, T, K - M, &b, &e);
  for (int s = M + b; s < M + e; ++s) n += status[s] == kTrackEmpty;
  return n;
}

// free slot of rank r (slot order) -> freelist[r], for the ranks below C (the candidates)
__device__ __forceinline__ void track_write_freelist(int t, int T, const unsigned char* __restrict__ status, int M, int K,
                                                     int rank, int C, int* __restrict__ freelist) {
  int b, e;
  track_range(t, T, K - M, &b, &e);
  for (int s = M + b; s < M + e && rank < C; ++s)
    if (status[s] == kTrackEmpty) freelist[rank++] = s;
}

// candidate of rank r (row-major cell order) -> BORN in slot freelist[r] at its seed point, for the ranks below Fr
__device__ __forceinline__ void track_assign(int t, int T, const double* __restrict__ lambda2,
                                             const unsigned char* __restrict__ cells, int G, double thr, int rank, int Fr,
                                             const int* __restrict__ freelist, float2* __restrict__ pos,
                                             unsigned char* __restrict__ status, int h, int Gx) {
  int b, e;
  track_range(t, T, G, &b, &e);
  for (int c = b; c < e && rank < Fr; ++c) {
    if (!track_candidate(lambda2, cells, c, thr)) continue;
    const int s = freelist[rank++];
    const int j = c / Gx, i = c - j * Gx;
    pos[s] = float2{(float)(i * h + h / 2), (float)(j * h + h / 2)};
    status[s] = kTrackBorn;
  }
}

#ifndef MFN_HOST_EMULATION
// exclusive scan of v over the CTA; *total = the sum.  Every thread of the CTA must call it.
__device__ __forceinline__ int track_block_scan(int v, int* total) {
  __shared__ int warp_sum[kTrackSeedThreads / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarp = blockDim.x >> 5;
  int x = v;
  for (int o = 1; o < 32; o <<= 1) {
    const int y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) warp_sum[warp] = x;
  __syncthreads();
  if (warp == 0) {
    int w = lane < nwarp ? warp_sum[lane] : 0;
    for (int o = 1; o < 32; o <<= 1) {
      const int y = __shfl_up_sync(0xffffffffu, w, o);
      if (lane >= o) w += y;
    }
    if (lane < nwarp) warp_sum[lane] = w;
  }
  __syncthreads();
  const int excl = x - v + (warp > 0 ? warp_sum[warp - 1] : 0);
  *total = warp_sum[nwarp - 1];
  __syncthreads();   // warp_sum is reused by the next call
  return excl;
}

// one CTA: the births of the frame *frame, then *frame += 1
__global__ void __launch_bounds__(kTrackSeedThreads)
    track_seed_kernel(const double* __restrict__ lambda2, const double* __restrict__ lambda_max,
                      const float* __restrict__ queries, int M, float2* __restrict__ pos, unsigned char* __restrict__ status,
                      unsigned char* __restrict__ cells, int* __restrict__ frame, int* __restrict__ dropped,
                      int* __restrict__ freelist, float2* __restrict__ out_pos, unsigned char* __restrict__ out_status,
                      int K, int H, int W, int h, int Gx, int Gy, float tau) {
  const int t = threadIdx.x, T = blockDim.x;
  const int f = *frame;
  const int G = Gx * Gy;
  track_seed_births(t, T, queries, M, f, pos, status, cells, H, W, h, Gx, Gy);
  __syncthreads();
  const double thr = (double)tau * *lambda_max;
  int C, Fr;
  const int c0 = track_block_scan(track_count_candidates(t, T, lambda2, cells, G, thr), &C);
  const int f0 = track_block_scan(track_count_free(t, T, status, M, K), &Fr);
  track_write_freelist(t, T, status, M, K, f0, C, freelist);
  __syncthreads();
  track_assign(t, T, lambda2, cells, G, thr, c0, Fr, freelist, pos, status, h, Gx);
  __syncthreads();
  if (out_pos)
    for (int s = t; s < K; s += T) {
      out_pos[s] = pos[s];
      out_status[s] = status[s];
    }
  if (t == 0) {
    *dropped = C > Fr ? C - Fr : 0;
    *frame = f + 1;
  }
}
#endif  // !MFN_HOST_EMULATION

}  // namespace mfn

#ifndef MFN_HOST_EMULATION
namespace {
bool track_finite_nonneg(float v) { return isfinite(v) && v >= 0.f; }
}  // namespace

extern "C" long long mfn_track_seed_workspace_bytes(int K) { return K > 0 ? 4LL * K : 0; }

extern "C" int mfn_track_texture(const unsigned char* frames, double* lambda2, double* lambda_max, int F, int H, int W,
                                 int spacing, void* stream) {
  using namespace mfn;
  MFN_REQUIRE(frames && lambda2 && lambda_max, MFN_ERR_INVALID_ARG, "mfn_track_texture: null pointer");
  MFN_REQUIRE(F > 0 && H > 0 && W > 0, MFN_ERR_INVALID_ARG, "mfn_track_texture: non-positive extent");
  MFN_REQUIRE(spacing >= 1, MFN_ERR_INVALID_ARG, "mfn_track_texture: spacing must be >= 1, got %d", spacing);
  MFN_REQUIRE(aligned(lambda2, 8) && aligned(lambda_max, 8), MFN_ERR_INVALID_ARG,
              "mfn_track_texture: lambda2 and lambda_max must be 8-byte aligned");
  MFN_REQUIRE((long long)H * W < (1LL << 31) && F <= 65535, MFN_ERR_ALIGNMENT,
              "mfn_track_texture: extents overflow kernel indexing");
  const int Gx = W / spacing, Gy = H / spacing, G = Gx * Gy;
  cudaStream_t st = as_stream(stream);
  const cudaError_t ce = cudaMemsetAsync(lambda_max, 0, sizeof(double) * F, st);
  if (ce != cudaSuccess) return fail((int)ce, "mfn_track_texture: cudaMemsetAsync: %s", cudaGetErrorString(ce));
  if (G == 0) return 0;   // the frame is narrower or lower than one cell: no seed points
  track_texture_kernel<<<dim3((G + 255) / 256, F), 256, 0, st>>>(
      frames, lambda2, reinterpret_cast<unsigned long long*>(lambda_max), H, W, spacing, Gx, G);
  return check_launch("track_texture_kernel");
}

extern "C" int mfn_track_advance(const float* flow_fw, const float* flow_bw, float* pos, unsigned char* status,
                                 unsigned char* cells, int K, int H, int W, int spacing, float alpha, float beta,
                                 float alpha_b, float beta_b, void* stream) {
  using namespace mfn;
  MFN_REQUIRE(flow_fw && flow_bw && pos && status && cells, MFN_ERR_INVALID_ARG, "mfn_track_advance: null pointer");
  MFN_REQUIRE(K > 0 && H > 0 && W > 0, MFN_ERR_INVALID_ARG, "mfn_track_advance: non-positive extent");
  MFN_REQUIRE(spacing >= 1, MFN_ERR_INVALID_ARG, "mfn_track_advance: spacing must be >= 1, got %d", spacing);
  MFN_REQUIRE(track_finite_nonneg(alpha) && track_finite_nonneg(beta) && track_finite_nonneg(alpha_b) &&
                  track_finite_nonneg(beta_b),
              MFN_ERR_INVALID_ARG, "mfn_track_advance: alpha, beta, alpha_b and beta_b must be finite and non-negative");
  MFN_REQUIRE(aligned(flow_fw, 8) && aligned(flow_bw, 8) && aligned(pos, 8), MFN_ERR_INVALID_ARG,
              "mfn_track_advance: flow_fw, flow_bw and pos must be 8-byte aligned");
  MFN_REQUIRE((long long)H * W < (1LL << 31), MFN_ERR_ALIGNMENT, "mfn_track_advance: extents overflow kernel indexing");
  const int Gx = W / spacing, Gy = H / spacing;
  cudaStream_t st = as_stream(stream);
  const cudaError_t ce = cudaMemsetAsync(cells, 0, (size_t)Gx * Gy, st);
  if (ce != cudaSuccess) return fail((int)ce, "mfn_track_advance: cudaMemsetAsync: %s", cudaGetErrorString(ce));
  track_advance_kernel<<<(K + 255) / 256, 256, 0, st>>>(
      reinterpret_cast<const float2*>(flow_fw), reinterpret_cast<const float2*>(flow_bw), reinterpret_cast<float2*>(pos),
      status, cells, K, H, W, spacing, Gx, Gy, alpha, beta, alpha_b, beta_b);
  return check_launch("track_advance_kernel");
}

extern "C" int mfn_track_seed(const double* lambda2, const double* lambda_max, const float* queries, int M, float* pos,
                              unsigned char* status, unsigned char* cells, int* frame, int* dropped, void* ws,
                              long long ws_bytes, float* out_pos, unsigned char* out_status, int K, int H, int W,
                              int spacing, float tau, void* stream) {
  using namespace mfn;
  MFN_REQUIRE(lambda2 && lambda_max && pos && status && cells && frame && dropped && ws && (queries || M == 0),
              MFN_ERR_INVALID_ARG, "mfn_track_seed: null pointer");
  MFN_REQUIRE(!out_pos == !out_status, MFN_ERR_INVALID_ARG, "mfn_track_seed: out_pos and out_status go together");
  MFN_REQUIRE(K > 0 && H > 0 && W > 0, MFN_ERR_INVALID_ARG, "mfn_track_seed: non-positive extent");
  MFN_REQUIRE(spacing >= 1, MFN_ERR_INVALID_ARG, "mfn_track_seed: spacing must be >= 1, got %d", spacing);
  MFN_REQUIRE(M >= 0 && M <= K, MFN_ERR_INVALID_ARG, "mfn_track_seed: %d queries for a capacity of %d slots", M, K);
  MFN_REQUIRE(track_finite_nonneg(tau), MFN_ERR_INVALID_ARG, "mfn_track_seed: tau must be finite and non-negative");
  MFN_REQUIRE(aligned(lambda2, 8) && aligned(lambda_max, 8) && aligned(pos, 8) && aligned(ws, 4) &&
                  (!out_pos || aligned(out_pos, 8)) && (!queries || aligned(queries, 4)),
              MFN_ERR_INVALID_ARG, "mfn_track_seed: lambda2, lambda_max, pos and out_pos must be 8-byte aligned, ws 4-byte");
  MFN_REQUIRE((long long)H * W < (1LL << 31), MFN_ERR_ALIGNMENT, "mfn_track_seed: extents overflow kernel indexing");
  const long long need = mfn_track_seed_workspace_bytes(K);
  MFN_REQUIRE(ws_bytes >= need, MFN_ERR_INVALID_ARG, "mfn_track_seed: workspace of %lld bytes, %lld needed", ws_bytes,
              need);
  track_seed_kernel<<<1, kTrackSeedThreads, 0, as_stream(stream)>>>(
      lambda2, lambda_max, queries, M, reinterpret_cast<float2*>(pos), status, cells, frame, dropped,
      static_cast<int*>(ws), reinterpret_cast<float2*>(out_pos), out_status, K, H, W, spacing, W / spacing, H / spacing,
      tau);
  return check_launch("track_seed_kernel");
}
#endif  // !MFN_HOST_EMULATION
