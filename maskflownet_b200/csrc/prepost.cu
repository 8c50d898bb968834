// prepost.cu -- the step either side of the network (SURVEY.md section 8f, row N3), fused:
//
//   mfn_preprocess_forward   replaces PipelineFlownet.predict / do_batch_mx (network/pipeline.py:206-212, 117-130):
//       img / 255  ->  centralize (subtract the per-sample RGB mean over BOTH images, :85-87)  ->  BilinearResize2D to the
//       padded size (multiples of 64, or `resize`)                     -- two launches (means, then resample) instead of ~8
//   mfn_postprocess_forward  replaces do_batch / predict (network/pipeline.py:134-143, 214-221):
//       Upsample(4)(flow2 * scale)  ->  BilinearResize2D back to the input size, times (H/H', W/W') per channel  ->
//       NCHW -> NHWC  ->  flip (y, x) -> (x, y)   (the layout predict.py writes to .flo)          -- one launch
//
// BilinearResize2D is MXNet's contrib operator [MXNet-recalled, bilinear_resize-inl.h]: "align corners" mapping
//   src = dst * (in - 1) / (out - 1),  i0 = (int)src,  i1 = i0 + (i0 < in - 1),  l = src - i0.
#include "common.cuh"

namespace mfn {

struct Lin {
  int i0, i1;
  float l;
};
__device__ __forceinline__ Lin resize_tap(int o, int n_in, int n_out) {
  Lin t;
  const float r = n_out > 1 ? (float)(n_in - 1) / (float)(n_out - 1) : 0.f;
  const float s = r * (float)o;
  t.i0 = (int)s;
  t.i1 = t.i0 + (t.i0 < n_in - 1 ? 1 : 0);
  t.l = s - (float)t.i0;
  return t;
}

template <typename T>
__global__ void __launch_bounds__(256)
    rgb_sum_kernel(const T* __restrict__ a, const T* __restrict__ b, float* __restrict__ sums, int planes, int HW, int slices) {
  // grid = planes * slices; partial sums of both images of plane p are added to sums[p]
  const int p = blockIdx.x / slices, s = blockIdx.x - p * slices;
  const long long beg = (long long)HW * s / slices, end = (long long)HW * (s + 1) / slices;
  const T* pa = a + (size_t)p * HW;
  const T* pb = b + (size_t)p * HW;
  float acc = 0.f;
  for (long long i = beg + threadIdx.x; i < end; i += blockDim.x) acc += (float)pa[i] + (float)pb[i];
  __shared__ float red[8];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x < 8) {
    float v = red[threadIdx.x];
#pragma unroll
    for (int o = 4; o > 0; o >>= 1) v += __shfl_xor_sync(0xffu, v, o);
    if (threadIdx.x == 0) atomicAdd(sums + p, v);
  }
}

template <typename T>
__global__ void __launch_bounds__(256)
    preprocess_kernel(const T* __restrict__ a, const T* __restrict__ b, const float* __restrict__ sums, float* __restrict__ oa,
                      float* __restrict__ ob, float* __restrict__ mean_out, int planes, int H, int W, int OH, int OW,
                      float in_scale) {
  const long long total = (long long)planes * OH * OW;
  const float inv_cnt = 1.f / (2.f * (float)H * (float)W);
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    const int ox = (int)(idx % OW), oy = (int)((idx / OW) % OH), p = (int)(idx / ((long long)OW * OH));
    const float mean = sums[p] * inv_cnt * in_scale;
    if (mean_out && ox == 0 && oy == 0) mean_out[p] = mean;
    const T* pa = a + (size_t)p * H * W;
    const T* pb = b + (size_t)p * H * W;
    float va, vb;
    if (OH == H && OW == W) {
      va = (float)pa[(size_t)oy * W + ox];
      vb = (float)pb[(size_t)oy * W + ox];
    } else {
      const Lin ty = resize_tap(oy, H, OH), tx = resize_tap(ox, W, OW);
      const float w00 = (1.f - ty.l) * (1.f - tx.l), w01 = (1.f - ty.l) * tx.l, w10 = ty.l * (1.f - tx.l), w11 = ty.l * tx.l;
      const size_t o00 = (size_t)ty.i0 * W + tx.i0, o01 = (size_t)ty.i0 * W + tx.i1, o10 = (size_t)ty.i1 * W + tx.i0,
                   o11 = (size_t)ty.i1 * W + tx.i1;
      va = w00 * (float)pa[o00] + w01 * (float)pa[o01] + w10 * (float)pa[o10] + w11 * (float)pa[o11];
      vb = w00 * (float)pb[o00] + w01 * (float)pb[o01] + w10 * (float)pb[o10] + w11 * (float)pb[o11];
    }
    oa[idx] = va * in_scale - mean;
    ob[idx] = vb * in_scale - mean;
  }
}

// out (N, H, W, CH) channels-last; channel k of the output = channel (flip ? CH-1-k : k) of the prediction, scaled by
// (H / 4Hq) for the y component and (W / 4Wq) for the x component when the size changes (flow only).
__global__ void __launch_bounds__(256)
    postprocess_kernel(const float* __restrict__ pred, float* __restrict__ out, int N, int CH, int Hq, int Wq, int H, int W,
                       int flip, int is_flow) {
  const int UH = 4 * Hq, UW = 4 * Wq;
  const long long total = (long long)N * H * W;
  const bool same = (UH == H && UW == W);
  const float sy = is_flow ? (float)H / (float)UH : 1.f, sx = is_flow ? (float)W / (float)UW : 1.f;
  for (long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (long long)gridDim.x * blockDim.x) {
    const int ox = (int)(idx % W), oy = (int)((idx / W) % H), n = (int)(idx / ((long long)W * H));
    for (int k = 0; k < CH; ++k) {
      const int c = flip ? CH - 1 - k : k;
      const float* pl = pred + ((size_t)n * CH + c) * Hq * Wq;
      float v;
      if (same) {
        v = upsample_at(pl, Hq, Wq, 4, oy, ox);
      } else {
        const Lin ty = resize_tap(oy, UH, H), tx = resize_tap(ox, UW, W);
        const float u00 = upsample_at(pl, Hq, Wq, 4, ty.i0, tx.i0), u01 = upsample_at(pl, Hq, Wq, 4, ty.i0, tx.i1);
        const float u10 = upsample_at(pl, Hq, Wq, 4, ty.i1, tx.i0), u11 = upsample_at(pl, Hq, Wq, 4, ty.i1, tx.i1);
        v = (1.f - ty.l) * ((1.f - tx.l) * u00 + tx.l * u01) + ty.l * ((1.f - tx.l) * u10 + tx.l * u11);
        if (is_flow) v *= (c == 0 ? sy : sx);      // prediction channel 0 = y, 1 = x (network/pipeline.py:105)
      }
      out[idx * CH + k] = v;
    }
  }
}

__global__ void scale_kernel(float* v, int n, float s) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) v[i] *= s;
}

static inline unsigned grid_of(long long total) {
  long long b = (total + 255) / 256;
  return (unsigned)(b < 1 ? 1 : (b > (long long)kNumSMs * 32 ? (long long)kNumSMs * 32 : b));
}

}  // namespace mfn

extern "C" int mfn_preprocess_forward(const void* img1, const void* img2, int is_uint8, float* out1, float* out2,
                                      float* rgb_mean, int N, int C, int H, int W, int OH, int OW, void* stream) {
  using namespace mfn;
  MFN_REQUIRE(img1 && img2 && out1 && out2 && rgb_mean, MFN_ERR_INVALID_ARG, "mfn_preprocess_forward: null pointer");
  MFN_REQUIRE(N > 0 && C > 0 && H > 0 && W > 0 && OH > 0 && OW > 0, MFN_ERR_INVALID_ARG,
              "mfn_preprocess_forward: non-positive extent");
  MFN_REQUIRE((long long)N * C * OH * OW < (1LL << 40) && (long long)H * W < (1LL << 31), MFN_ERR_ALIGNMENT,
              "mfn_preprocess_forward: extents overflow kernel indexing");
  cudaStream_t st = as_stream(stream);
  const int planes = N * C;
  cudaError_t ce = cudaMemsetAsync(rgb_mean, 0, sizeof(float) * planes, st);
  if (ce != cudaSuccess) return fail((int)ce, "mfn_preprocess_forward: cudaMemsetAsync: %s", cudaGetErrorString(ce));
  int slices = (kNumSMs * 4 + planes - 1) / planes;
  if (slices < 1) slices = 1;
  // rgb_mean first accumulates the per-plane sums (atomics over `slices` partial sums), is read as such by the resampling
  // kernel, and is turned into the means by a last tiny launch
  if (is_uint8)
    rgb_sum_kernel<unsigned char><<<planes * slices, 256, 0, st>>>(static_cast<const unsigned char*>(img1),
                                                                  static_cast<const unsigned char*>(img2), rgb_mean, planes,
                                                                  H * W, slices);
  else
    rgb_sum_kernel<float><<<planes * slices, 256, 0, st>>>(static_cast<const float*>(img1), static_cast<const float*>(img2),
                                                          rgb_mean, planes, H * W, slices);
  int rc = check_launch("rgb_sum_kernel");
  if (rc) return rc;
  const long long total = (long long)planes * OH * OW;
  const float in_scale = is_uint8 ? 1.f / 255.f : 1.f;
  if (is_uint8)
    preprocess_kernel<unsigned char><<<grid_of(total), 256, 0, st>>>(static_cast<const unsigned char*>(img1),
                                                                    static_cast<const unsigned char*>(img2), rgb_mean, out1,
                                                                    out2, nullptr, planes, H, W, OH, OW, in_scale);
  else
    preprocess_kernel<float><<<grid_of(total), 256, 0, st>>>(static_cast<const float*>(img1), static_cast<const float*>(img2),
                                                            rgb_mean, out1, out2, nullptr, planes, H, W, OH, OW, in_scale);
  rc = check_launch("preprocess_kernel");
  if (rc) return rc;
  scale_kernel<<<(planes + 255) / 256, 256, 0, st>>>(rgb_mean, planes, in_scale / (2.f * (float)H * (float)W));
  return check_launch("preprocess_kernel");
}

extern "C" int mfn_postprocess_forward(const float* pred, float* out, int N, int channels, int Hq, int Wq, int H, int W,
                                       int flip_channels, int is_flow, void* stream) {
  using namespace mfn;
  MFN_REQUIRE(pred && out, MFN_ERR_INVALID_ARG, "mfn_postprocess_forward: null pointer");
  MFN_REQUIRE(N > 0 && channels > 0 && channels <= 4 && Hq > 0 && Wq > 0 && H > 0 && W > 0, MFN_ERR_INVALID_ARG,
              "mfn_postprocess_forward: bad extent");
  MFN_REQUIRE(!is_flow || channels == 2, MFN_ERR_INVALID_ARG, "mfn_postprocess_forward: a flow has 2 channels");
  postprocess_kernel<<<grid_of((long long)N * H * W), 256, 0, as_stream(stream)>>>(pred, out, N, channels, Hq, Wq, H, W,
                                                                                 flip_channels ? 1 : 0, is_flow ? 1 : 0);
  return check_launch("postprocess_kernel");
}
