// warp_lin.cu -- K3 (flow-guided deformable warp x occlusion mask) evaluated EXACTLY through linearity, for every pixel and
// both border rules; no per-pixel fallback list, cost independent of the flow field.
//
// Reference semantics: network/MaskFlownet.py:228-233 -> network/layer.py:117-124 (DeformableConvolution, 3x3, all nine tap
// offsets equal to the up-sampled flow), then * sigmoid(mask) + trade-off -> LeakyReLU.
//
// Every tap samples x at (h_i, w_j) = (y - 1 + i + dy, x - 1 + j + dx) with a SEPARABLE rule: the sample is a(h_i)^T X b(w_j),
// where the per-axis coefficient vector is
//   zero-corner rule (DCNv2 / torchvision, MFN_BORDER_ZERO_CORNER):  a = a_Z = the hat function on the zero-extended axis;
//   MXNet-1.5 rule (MFN_BORDER_MXNET15):  a = a_Z + a_D with a_D(h) = -(1 + h) e_0       for h in (-1, 0)   (sample forced to 0)
//                                                            a_D(h) = (h - (n-1)) e_{n-1} for h in (n-1, n) (collapsed on the last pixel)
//                                                            a_D(h) = 0 elsewhere.
// Summing over the taps with the weights W_ij:
//   Z x Z : bilinear sample at (y + dy, x + dx) of Yext = conv3x3(x, W) evaluated on the grid extended by one pixel per side
//           (wgmma kernel, conv3x3_wgmma.cu with ext = 1) -- all of the operator in zero-corner mode;
//   D x Z : sum_i alpha_i * lerp_w( Rrow[B_i][i] )   with Rrow[B][i] = conv1d(x[row B], W[i, :]) on the extended row,
//   Z x D : sum_j beta_j  * lerp_h( Rcol[B_j][j] )   with Rcol[B][j] = conv1d(x[:, col B], W[:, j]),
//   D x D : sum_ij alpha_i beta_j T[B_i][B_j][i][j]  with T = W_ij . x[:, row B_i, col B_j]
// (B = first / last row or column).  The three tables come out of the SAME tensor-core convolution: in its ext = 2 mode
// the kernel reads a virtual image whose rows / columns n .. n+5 are [0, 0, first, 0, 0, last], so the isolated copies of
// the border rows / columns / corner pixels produce exactly Rrow, Rcol and T next to Yext (one launch, ~10-40 % more
// tiles).  Only pixels whose taps reach the one-pixel bands read them.  Band membership uses the same float expression (y - 1 + i) + dy as the reference kernel, so the operator's
// discontinuities (h = 0, h = H) are taken on the same side as the tap-by-tap kernels and the oracle.
#include "mma_tiles.cuh"

namespace mfn {
namespace wl {

struct Band {
  float a[3];   // correction coefficient of tap row / column i (0 = not in a band)
  int B[3];     // 0 = first row / column, 1 = last
  bool any;
};
__device__ __forceinline__ Band bands(int p, float d, int n) {
  Band b;
  b.any = false;
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    const float h = (float)(p - 1 + i) + d;
    float a = 0.f;
    int B = 0;
    if (h > -1.f && h < 0.f) {
      a = -(1.f + h);
    } else if (h > (float)(n - 1) && h < (float)n) {
      a = h - (float)(n - 1);
      B = 1;
    }
    b.a[i] = a;
    b.B[i] = B;
    b.any = b.any || (a != 0.f);
  }
  return b;
}

// Yall = conv3x3_wgmma(ext = 2): (N, F, H + 8, W + 8); entry (r, v) <-> position (r - 1, v - 1) of the virtual image
//   rows 0 .. H+1, cols 0 .. W+1   Yext (the extended convolution)
//   rows H+4-i / H+7-i             the 1-D convolution of the first / last image row with weight row i   (Rrow)
//   cols W+4-j / W+7-j             ... of the first / last image column with weight column j               (Rcol)
//   their intersections            W_ij . x[corner]                                                         (T)
// One thread per (pixel, chunk of FCH output channels): all accesses coalesced along x.
constexpr int FCH = 16;   // smallest channel chunk (a multiple of the 8-channel load batch); the launch picks 16 / 32 / 64 per thread
template <int BORDER>
__global__ void __launch_bounds__(256)
    warp_lin_kernel(const float* __restrict__ Yall, const float* __restrict__ flow_c, const float* __restrict__ mask_c,
                    const float* __restrict__ bias, const float* __restrict__ tradeoff, float* __restrict__ out,
                    float* __restrict__ flow_up_out, float* __restrict__ mask_up_out, int N, int H, int W, int F, int up,
                    float flow_scale, float level_stride, float slope, int grow, int fch) {
  const long long total = (long long)N * H * W;
  const size_t plane = (size_t)H * W;
  const int WA = W + grow, HA = H + grow;
  const size_t aplane = (size_t)HA * WA;
  // per-pixel set-up (flow / mask up-sampling, corner weights, band entries) is ~40 % of a 16-channel thread's
  // instructions: big levels take more channels per thread (fch), small levels keep 16 for the sake of parallelism
  const int f0 = blockIdx.y * fch, f1 = min(F, f0 + fch);
  const int Hc = H / up, Wc = W / up;
  for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < total; p += (long long)gridDim.x * blockDim.x) {
    const unsigned pu = (unsigned)p;                   // total < 2^31 (checked by the host): 32-bit index arithmetic
    const int n = (int)(pu / (unsigned)plane), rem = (int)(pu - (unsigned)n * (unsigned)plane);
    const int y = rem / W, xq = rem - y * W;
    const float* fc = flow_c + (size_t)n * 2 * Hc * Wc;
    float fy, fx, mask_v;
    if (up == 2) {                                     // the network's Upsample(2): constant-folded taps
      fy = upsample_at(fc, Hc, Wc, 2, y, xq);
      fx = upsample_at(fc + (size_t)Hc * Wc, Hc, Wc, 2, y, xq);
      mask_v = mask_c ? upsample_at(mask_c + (size_t)n * Hc * Wc, Hc, Wc, 2, y, xq) : 0.f;
    } else {
      fy = upsample_at(fc, Hc, Wc, up, y, xq);
      fx = upsample_at(fc + (size_t)Hc * Wc, Hc, Wc, up, y, xq);
      mask_v = mask_c ? upsample_at(mask_c + (size_t)n * Hc * Wc, Hc, Wc, up, y, xq) : 0.f;
    }
    const size_t pix = (size_t)y * W + xq;
    if (blockIdx.y == 0) {
      if (flow_up_out) {
        flow_up_out[((size_t)n * 2 + 0) * plane + pix] = fy;
        flow_up_out[((size_t)n * 2 + 1) * plane + pix] = fx;
      }
      if (mask_up_out && mask_c) mask_up_out[(size_t)n * plane + pix] = mask_v;
    }
    // offsets exactly as the reference rounds them: (flow * scale) / stride   (MaskFlownet.py:230)
    const float dy = __fdiv_rn(__fmul_rn(fy, flow_scale), level_stride);
    const float dx = __fdiv_rn(__fmul_rn(fx, flow_scale), level_stride);
    const float h0 = (float)y + dy, w0 = (float)xq + dx;
    // ---- Z x Z: bilinear sample of the extended convolution ----
    const float fh = floorf(h0), fw = floorf(w0);
    const bool farout = !(h0 > -3.f && h0 < (float)(H + 2) && w0 > -3.f && w0 < (float)(W + 2));   // keeps the int conversion defined
    const int i0 = farout ? -8 : (int)fh + 1, j0 = farout ? -8 : (int)fw + 1;
    const float lh = h0 - fh, lw = w0 - fw;
    const bool r0 = i0 >= 0 && i0 <= H + 1, r1 = i0 + 1 >= 0 && i0 + 1 <= H + 1;
    const bool c0 = j0 >= 0 && j0 <= W + 1, c1 = j0 + 1 >= 0 && j0 + 1 <= W + 1;
    const float w00 = (r0 && c0) ? (1.f - lh) * (1.f - lw) : 0.f, w01 = (r0 && c1) ? (1.f - lh) * lw : 0.f;
    const float w10 = (r1 && c0) ? lh * (1.f - lw) : 0.f, w11 = (r1 && c1) ? lh * lw : 0.f;
    const int ic0 = min(max(i0, 0), H + 1), ic1 = min(max(i0 + 1, 0), H + 1);
    const int jc0 = min(max(j0, 0), W + 1), jc1 = min(max(j0 + 1, 0), W + 1);
    const int o00 = ic0 * WA + jc0, o01 = ic0 * WA + jc1, o10 = ic1 * WA + jc0, o11 = ic1 * WA + jc1;
    const bool anyz = (w00 != 0.f) || (w01 != 0.f) || (w10 != 0.f) || (w11 != 0.f);
    Band bh, bw;
    bh.any = bw.any = false;
    if (BORDER == MFN_BORDER_MXNET15) {
      bh = bands(y, dy, H);
      bw = bands(xq, dx, W);
    }
    const float sig = mask_c ? sigmoidf_(mask_v) : 1.f;
    const float* yp = Yall + ((size_t)n * F + f0) * aplane;
    float* op = out + ((size_t)n * F + f0) * plane + pix;
    const float* tp = tradeoff ? tradeoff + ((size_t)n * F + f0) * plane + pix : nullptr;
    // ---- MXNet-1.5 band terms as (offset, weight) pairs, computed ONCE per pixel: at most one tap row and one tap column
    //      can sit in a band (bands are one pixel wide, taps one pixel apart, H, W >= 4): D x Z -> two entries along the
    //      band row's 1-D convolution, Z x D -> two along the band column's, D x D -> the corner product
    int eo[5] = {0, 0, 0, 0, 0};
    float ew[5] = {0.f, 0.f, 0.f, 0.f, 0.f};
    if (BORDER == MFN_BORDER_MXNET15) {
      float a = 0.f, b = 0.f;
      int rI = 0, cJ = 0;
#pragma unroll
      for (int i = 0; i < 3; ++i)
        if (bh.a[i] != 0.f) {
          a = bh.a[i];
          rI = H + 4 + 3 * bh.B[i] - i;
        }
#pragma unroll
      for (int j = 0; j < 3; ++j)
        if (bw.a[j] != 0.f) {
          b = bw.a[j];
          cJ = W + 4 + 3 * bw.B[j] - j;
        }
      eo[0] = rI * WA + jc0;
      ew[0] = c0 ? a * (1.f - lw) : 0.f;
      eo[1] = rI * WA + jc1;
      ew[1] = c1 ? a * lw : 0.f;
      eo[2] = ic0 * WA + cJ;
      ew[2] = r0 ? b * (1.f - lh) : 0.f;
      eo[3] = ic1 * WA + cJ;
      ew[3] = r1 ? b * lh : 0.f;
      eo[4] = rI * WA + cJ;
      ew[4] = a * b;
    }
    const bool warp_bands = BORDER == MFN_BORDER_MXNET15 && __any_sync(__activemask(), bh.any || bw.any);
    // branch-free channel loop: the corner offsets are clamped into the array and the weights of out-of-range corners are
    // zero, so every load is legal and the loads of eight channels are issued before the first use (per-channel band tests
    // multiplied the instructions per channel)
    const int nf = f1 - f0;
#pragma unroll 1
    for (int fb = 0; fb < nf; fb += 8) {
      float v[8], tv[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        const bool on = fb + u < nf;
        const float* q = yp + (size_t)(on ? fb + u : 0) * aplane;
        v[u] = w00 * __ldg(q + o00) + w01 * __ldg(q + o01) + w10 * __ldg(q + o10) + w11 * __ldg(q + o11);
        tv[u] = (tp && on) ? __ldg(tp + (size_t)(fb + u) * plane) : 0.f;
      }
      if (warp_bands) {
#pragma unroll
        for (int u = 0; u < 8; ++u) {
          const float* q = yp + (size_t)(fb + u < nf ? fb + u : 0) * aplane;
          v[u] += ew[0] * __ldg(q + eo[0]) + ew[1] * __ldg(q + eo[1]) + ew[2] * __ldg(q + eo[2]) + ew[3] * __ldg(q + eo[3]) +
                  ew[4] * __ldg(q + eo[4]);
        }
      }
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        if (fb + u < nf) {
          float r = v[u];
          if (bias) r += __ldg(bias + f0 + fb + u);
          r = r * sig + tv[u];
          op[(size_t)(fb + u) * plane] = leaky(r, slope);
        }
      }
    }
  }
}

}  // namespace wl

long long warp_lin_workspace_bytes(int N, int F, int H, int W) { return (long long)N * F * (H + 8) * (W + 8) * 4 + 64; }

// returns -1 when the extended wgmma convolution does not fit the shape (caller uses the list-based path)
int launch_warp_lin(const float* x, const float* flow_c, const float* mask_c, const float* weight, const void* packed_weight,
                    const float* bias, const float* tradeoff, void* workspace, float* out, float* fup, float* mup, int N,
                    int C, int H, int W, int F, int up, float fs, float ls, float slope, int border_mode, cudaStream_t st) {
  using namespace wl;
  (void)weight;
  float* Yall = static_cast<float*>(workspace);
  const unsigned char* wp = static_cast<const unsigned char*>(packed_weight);
  // zero-corner rule: the extended convolution alone (grid + 1 pixel per side); MXNet-1.5 rule: + the band rows / columns
  const int ext = border_mode == MFN_BORDER_MXNET15 ? 2 : 1, grow = ext == 2 ? 8 : 2;
  int rc = conv3x3_wgmma_launch(x, (long long)C * H * W, wp + conv3x3_sync_packed_bytes(C, F), nullptr, Yall,
                               (long long)F * (H + grow) * (W + grow), N, C, H, W, F, 1, 1, MFN_CONV_OUT_NCHW, 1.0f, st, ext);
  if (rc) return rc;
  const long long total = (long long)N * H * W;
  if (total >= (1LL << 31)) return -1;
  long long blocks = (total + 255) / 256;
  if (blocks > (long long)kNumSMs * 8) blocks = (long long)kNumSMs * 8;
  // channels per thread: doubled while at least one resident wave of threads (one per SM x 512) remains
  int fch = FCH;
  while (fch < 64 && fch < F && total * ((F + 2 * fch - 1) / (2 * fch)) >= (long long)kNumSMs * 512) fch *= 2;
  const dim3 grid((unsigned)blocks, (unsigned)((F + fch - 1) / fch));
  if (border_mode == MFN_BORDER_MXNET15)
    warp_lin_kernel<MFN_BORDER_MXNET15><<<grid, 256, 0, st>>>(Yall, flow_c, mask_c, bias, tradeoff, out, fup, mup, N, H, W, F, up,
                                                             fs, ls, slope, grow, fch);
  else
    warp_lin_kernel<MFN_BORDER_ZERO_CORNER><<<grid, 256, 0, st>>>(Yall, flow_c, mask_c, bias, tradeoff, out, fup, mup, N, H, W, F,
                                                                 up, fs, ls, slope, grow, fch);
  return check_launch("warp_lin_kernel");
}

}  // namespace mfn
