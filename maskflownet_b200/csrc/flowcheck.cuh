// flowcheck.cuh -- the forward-backward check of Sundaram, Brox and Keutzer (ECCV 2010) at a float position: the flow of
// one direction sampled bilinearly at a target, and the round-trip test against it.  Shared by mfn_flow_consistency
// (consistency.cu: targets of integer pixels) and the point tracker (track.cu: targets of subpixel track positions), so
// both apply the same corner rule and the same arithmetic.
#pragma once

namespace mfn {

__device__ __forceinline__ float fb_lerp(float p, float q, float w) { return p * (1.f - w) + q * w; }

// The H x W flow plane sampled bilinearly at (qx, qy), which must lie inside [0, W-1] x [0, H-1]: corners x0 = floor(qx),
// x1 = min(x0 + 1, W - 1), the same in y, weights q - floor(q).  Every read is inside the plane.
__device__ __forceinline__ float2 fb_sample(const float2* __restrict__ plane, int H, int W, float qx, float qy) {
  const int x0 = (int)floorf(qx), y0 = (int)floorf(qy);
  const int x1 = min(x0 + 1, W - 1), y1 = min(y0 + 1, H - 1);
  const float wx = qx - (float)x0, wy = qy - (float)y0;
  const float2 a = __ldg(plane + (size_t)y0 * W + x0), b = __ldg(plane + (size_t)y0 * W + x1);
  const float2 c = __ldg(plane + (size_t)y1 * W + x0), d = __ldg(plane + (size_t)y1 * W + x1);
  return float2{fb_lerp(fb_lerp(a.x, b.x, wx), fb_lerp(c.x, d.x, wx), wy),
                fb_lerp(fb_lerp(a.y, b.y, wx), fb_lerp(c.y, d.y, wx), wy)};
}

// true where the round trip of uv and the other direction's flow b at its target cancels:
// |uv + b|^2 <= alpha (|uv|^2 + |b|^2) + beta with a finite right-hand side.  NaN or inf anywhere gives false.
__device__ __forceinline__ bool fb_consistent(float2 uv, float2 b, float alpha, float beta) {
  const float su = uv.x + b.x, sv = uv.y + b.y;
  const float d2 = su * su + sv * sv;
  const float m2 = uv.x * uv.x + uv.y * uv.y + b.x * b.x + b.y * b.y;
  const float rhs = alpha * m2 + beta;
  return d2 <= rhs && rhs <= 3.402823466e38f;   // rhs <= FLT_MAX: finite
}

// 1 where the pixel (x, y) with flow uv has no consistent match in `other` (the H x W flow plane of the other direction):
// its target (x+u, y+v) lies outside [0, W-1] x [0, H-1] (NaN included), or fb_consistent fails at the target (an inf
// corner reaches the sample as inf, or as NaN where its weight is 0: both give 1).
__device__ __forceinline__ unsigned char fb_occluded(const float2* __restrict__ other, int H, int W, int x, int y,
                                                     float2 uv, float alpha, float beta) {
  const float qx = (float)x + uv.x, qy = (float)y + uv.y;
  if (!(qx >= 0.f && qx <= (float)(W - 1) && qy >= 0.f && qy <= (float)(H - 1))) return 1;
  return fb_consistent(uv, fb_sample(other, H, W, qx, qy), alpha, beta) ? 0 : 1;
}

}  // namespace mfn
