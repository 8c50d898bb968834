/*
 * maskflow_b200.h -- C ABI of libmaskflow_b200.so: the MaskFlownet hot path on NVIDIA H100 (sm_90a).
 *
 * The reference (microsoft/MaskFlownet) reaches this path through Apache MXNet's operator registry
 * (the `F` namespace handed to HybridBlock.hybrid_forward).  Each entry point below replaces one MXNet
 * operator call site of the reference, or a fused group of them; the citation after "replaces:" is the
 * reference file:line (under /root/reference) whose call it serves.
 *
 * Conventions (SURVEY.md section 8b)
 *   - extern "C", plain pointers and ints only.  No C++ / torch types cross this boundary.
 *   - Every tensor is fp32, NCHW, contiguous unless a stride argument says otherwise; all pointers are
 *     DEVICE pointers owned by the caller.  The library never allocates or frees device memory and
 *     keeps no pointer after a call returns.
 *   - Every call is asynchronous: kernels are enqueued on `stream` (a cudaStream_t passed as void*; NULL =
 *     the legacy default stream) of the caller's current device.  No host synchronisation happens inside.
 *   - Return value: 0 = ok; < 0 = MFN_ERR_* (argument / support error, nothing was launched);
 *     > 0 = a cudaError_t raised by the launch.  mfn_last_error() returns a thread-local message.
 *   - Flow tensors follow the reference: 2 channels ordered (y, x) (network/pipeline.py:105),
 *     in units of pixels/scale at full resolution (self.scale = 20, network/MaskFlownet.py:69).
 */
#ifndef MASKFLOW_B200_H_
#define MASKFLOW_B200_H_

#ifdef __cplusplus
extern "C" {
#endif

#define MFN_VERSION 100 /* 0.1.0 */

#if defined(__GNUC__)
#define MFN_API __attribute__((visibility("default")))
#else
#define MFN_API
#endif

#define MFN_OK 0
#define MFN_ERR_INVALID_ARG (-1) /* null pointer, non-positive extent, inconsistent shapes           */
#define MFN_ERR_UNSUPPORTED (-2) /* parameter combination outside what the kernels implement         */
#define MFN_ERR_ALIGNMENT (-3)   /* pointer not 4-byte aligned / extents overflow 32-bit indexing    */

/* Correlation algorithm selector (mfn_correlation_forward `algo`). */
#define MFN_CORR_AUTO 0       /* pick per shape: MMA when kernel_size=1,strides=1,multiply; else GENERIC */
#define MFN_CORR_GENERIC 1    /* every MXNet parameter combination, one thread per output, exact fp32 */
#define MFN_CORR_SIMT 2       /* tiled fp32 FMA kernel, exact fp32 accumulation (k=1, strides=1, multiply) */
#define MFN_CORR_MMA_BF16X3 3 /* tensor-core kernel: bf16 hi/lo split, 3 MMAs per product, fp32 accumulate */

/* Deformable-convolution border rule (SURVEY.md section 8c). */
#define MFN_BORDER_MXNET15 0    /* zero unless 0<=h<H, 0<=w<W; floor>=size-1 collapses on the last pixel */
#define MFN_BORDER_ZERO_CORNER 1 /* DCNv2 / torchvision: h>-1, w>-1; corners outside contribute zero    */

MFN_API int mfn_version(void);
MFN_API const char* mfn_last_error(void);
/* Name of the kernel variant the last successful call on this thread launched (diagnostics / tests). */
MFN_API const char* mfn_last_kernel(void);
/* Number of kernel launches issued by this library since load (process-wide, monotonically increasing). */
MFN_API unsigned long long mfn_launch_count(void);
/* Process-wide tuning / test knobs.  Keys: "corr_grid_cap" (>0 caps the persistent grid of the tensor-core correlation
 * kernels; tests use it to force long per-CTA tile runs), "corr_disable_ring" (1 = never pick the strip-marching kernel). */
MFN_API int mfn_set_tuning(const char* key, int value);

/* ---------------------------------------------------------------------------------------------------
 * Correlation cost volume.
 * replaces: F.Correlation(data1, data2, pad_size, kernel_size, max_displacement, stride1, stride2,
 *           is_multiply)  -- network/MaskFlownet.py:193-195 (md=4, 81 ch) and :440-441 (md=2, 25 ch),
 *           plus the LeakyReLU(0.1) that always follows it (:217,235,253,271,289; :467-529) when
 *           leaky_slope != 1.
 *   out[n,q,i,j] = act( 1/(k*k*C) * sum_{h,w<k} sum_c d1p[n,c,y1+h,x1+w] (*) d2p[n,c,y2+h,x2+w] )
 *   with d*p the inputs zero-padded by pad_size, (x1,y1)=(j*stride1+md, i*stride1+md),
 *   (x2,y2)=(x1+(q%G-r)*stride2, y1+(q/G-r)*stride2), r=md/stride2, G=2r+1, (*) = product (is_multiply)
 *   or |a-b|.  Output extents: D=G*G, OH=ceil((H+2*pad-2*(md+(k-1)/2))/stride1), OW likewise.
 * out_batch_stride: elements between consecutive samples of `out` (0 = D*OH*OW); lets the caller point
 *   `out` at channel 0 of a wider pre-allocated concat buffer (network/MaskFlownet.py:236).
 * act(v) = v > 0 ? v : leaky_slope * v   (leaky_slope = 1 disables it).
 * ------------------------------------------------------------------------------------------------- */
MFN_API int mfn_correlation_forward(const float* data1, const float* data2, float* out, int N, int C, int H,
                            int W, int pad_size, int kernel_size, int max_displacement, int stride1,
                            int stride2, int is_multiply, long long out_batch_stride,
                            float leaky_slope, int algo, void* stream);

/* Backward of the above for the regime the reference uses (kernel_size=1, strides 1, multiply,
 * pad_size == max_displacement).  replaces: the implicit autograd of F.Correlation under
 * autograd.record() -- network/pipeline.py:97,112-113.
 *   g1[n,c,y,x] = 1/C sum_q go'[n,q,y,x]       * d2[n,c,y+dy,x+dx]
 *   g2[n,c,y,x] = 1/C sum_q go'[n,q,y-dy,x-dx] * d1[n,c,y-dy,x-dx]
 * If `out` (the forward result, post-activation) is non-NULL, go' = go * (out>0 ? 1 : leaky_slope),
 * i.e. the LeakyReLU backward is fused; otherwise go' = go.  grad_out/out share out_batch_stride. */
MFN_API int mfn_correlation_backward(const float* grad_out, const float* out, const float* data1,
                             const float* data2, float* grad1, float* grad2, int N, int C, int H,
                             int W, int max_displacement, long long out_batch_stride,
                             float leaky_slope, void* stream);

/* ---------------------------------------------------------------------------------------------------
 * Deformable convolution (signature-faithful form).
 * replaces: F.contrib.DeformableConvolution(data, offset, weight[, bias], kernel, stride, dilate, pad,
 *           num_filter, num_group, no_bias, layout, num_deformable_group) -- network/layer.py:117-124
 *           with the kwargs of layer.py:91-95.
 * Implemented: kernel 3x3, stride 1, dilate 1, pad 1, num_group 1, num_deformable_group 1 (the only
 * configuration the reference instantiates, network/MaskFlownet.py:155-158, 403-407); anything else
 * returns MFN_ERR_UNSUPPORTED.  offset is (N,18,H,W): channel 2k = dy, 2k+1 = dx of tap k = i*3+j.
 * bias may be NULL (no_bias).
 * ------------------------------------------------------------------------------------------------- */
MFN_API int mfn_deformable_conv_forward(const float* data, const float* offset, const float* weight,
                                const float* bias, float* out, int N, int C, int H, int W, int F,
                                int kernel_h, int kernel_w, int stride_h, int stride_w, int dilate_h,
                                int dilate_w, int pad_h, int pad_w, int num_group,
                                int num_deformable_group, int border_mode, void* stream);

/* Backward of mfn_deformable_conv_forward (analytic derivative of the forward as defined above).
 * grad_data / grad_offset / grad_weight / grad_bias may each be NULL (not computed).  grad_data,
 * grad_weight and grad_bias are ACCUMULATED INTO (atomics): the caller zero-fills them first. */
MFN_API int mfn_deformable_conv_backward(const float* grad_out, const float* data, const float* offset,
                                 const float* weight, float* grad_data, float* grad_offset,
                                 float* grad_weight, float* grad_bias, int N, int C, int H, int W,
                                 int F, int border_mode, void* stream);

/* ---------------------------------------------------------------------------------------------------
 * Fused flow-guided feature warp of one pyramid level.
 * replaces, for level L of the S head (network/MaskFlownet.py:228-233; same at :246-251,264-269,282-287):
 *     flowL = Upsample(2)(flow_{L+1}); maskL = Upsample(2)(mask_{L+1})
 *     warpL = deformL(c2L, repeat(flowL*scale/strideL, 9))                  (layer.py:117-124)
 *     warpL = LeakyReLU( warpL * sigmoid(maskL) + convLf(featL) )
 * and for the cascade (network/MaskFlownet.py:463-466, 479-481, ...): the same without mask / trade-off.
 *   x            (N,C,H,W)      features to warp (c2L)
 *   flow_coarse  (N,2,Hc,Wc)    (y,x) flow; Hc=H/up, Wc=W/up with up = upsample_factor (1 or 2)
 *   mask_coarse  (N,1,Hc,Wc)    occlusion-mask logits or NULL
 *   weight (F,C,3,3), bias (F) or NULL, tradeoff (N,F,H,W) or NULL (already-computed convLf output)
 *   out          (N,F,H,W)      LeakyReLU_{leaky_slope}( (conv + bias) * sigmoid(mask) + tradeoff )
 *   flow_up_out  (N,2,H,W) or NULL, mask_up_out (N,1,H,W) or NULL: the up-sampled flow / mask, which the
 *                reference also feeds to the decoder (MaskFlownet.py:236)
 *   conv_out     (N,F,H,W) or NULL: conv + bias before the mask multiply (saved for backward)
 * flow offsets are computed as (flow_up * flow_scale) / level_stride, rounded like the reference.
 * ------------------------------------------------------------------------------------------------- */
MFN_API int mfn_warp_mask_forward(const float* x, const float* flow_coarse, const float* mask_coarse,
                          const float* weight, const float* bias, const float* tradeoff, float* out,
                          float* flow_up_out, float* mask_up_out, float* conv_out, int N, int C,
                          int H, int W, int F, int upsample_factor, float flow_scale,
                          float level_stride, float leaky_slope, int border_mode, void* stream);

/* Tensor-core variant of mfn_warp_mask_forward (same arguments and results; fp32-accurate bf16x3 arithmetic): `weight` is
 * replaced by the packed image of the (F,C,3,3) deformable-convolution weight produced by mfn_conv3x3_pack_weights
 * (mfn_conv3x3_packed_bytes(C, F) bytes).  F <= 128.  Inference path (no saved tensors needed beyond conv_out). */
MFN_API int mfn_warp_mask_forward_tc(const float* x, const float* flow_coarse, const float* mask_coarse,
                                     const void* packed_weight, const float* bias, const float* tradeoff, float* out,
                                     float* flow_up_out, float* mask_up_out, float* conv_out, int N, int C, int H, int W,
                                     int F, int upsample_factor, float flow_scale, float level_stride, float leaky_slope,
                                     int border_mode, void* stream);

/* Same operator through linearity (inference): because all nine taps share one offset per pixel, the deformable
 * convolution equals bilinear re-sampling of the PLAIN 3x3 convolution Y = conv(x, weight) wherever the nine samples fall
 * inside the image.  Three launches: Y on the tensor cores (packed_weight = mfn_conv3x3_pack_weights(weight)), the fused
 * re-sampling epilogue, and the tap-by-tap kernel over the list of pixels whose warped centre is within two pixels of the
 * border (where MFN_BORDER_* rules are not linear).  workspace: caller-owned, mfn_warp_resample_workspace_bytes() bytes,
 * 16-byte aligned.  Results equal mfn_warp_mask_forward up to fp32 rounding (tests: 1e-4). */
MFN_API long long mfn_warp_resample_workspace_bytes(int N, int F, int H, int W);
MFN_API int mfn_warp_mask_forward_resample(const float* x, const float* flow_coarse, const float* mask_coarse,
                                           const float* weight, const void* packed_weight, const float* bias,
                                           const float* tradeoff, void* workspace, float* out, float* flow_up_out,
                                           float* mask_up_out, int N, int C, int H, int W, int F, int upsample_factor,
                                           float flow_scale, float level_stride, float leaky_slope, int border_mode,
                                           void* stream);

/* Backward of mfn_warp_mask_forward.
 *   in : grad_out (N,F,H,W); out (forward result); conv_out (saved); x; flow_up (N,2,H,W, the forward's
 *        flow_up_out); mask_up (N,1,H,W) or NULL; weight
 *   out: grad_x (N,C,H,W, accumulated: zero-fill first), grad_flow_up (N,2,H,W, overwritten: gradient
 *        w.r.t. the UP-SAMPLED flow through the offsets only), grad_mask_up (N,1,H,W, overwritten) or NULL,
 *        grad_weight (F,C,3,3) / grad_bias (F) (accumulated), grad_tradeoff (N,F,H,W, overwritten) or NULL.
 * The transposed Upsample(2) of grad_flow_up / grad_mask_up is mfn_upsample_backward. */
MFN_API int mfn_warp_mask_backward(const float* grad_out, const float* out, const float* conv_out,
                           const float* x, const float* flow_up, const float* mask_up,
                           const float* weight, float* grad_x, float* grad_flow_up,
                           float* grad_mask_up, float* grad_weight, float* grad_bias,
                           float* grad_tradeoff, float* grad_conv_ws, int N, int C, int H, int W,
                           int F, float flow_scale, float level_stride, float leaky_slope,
                           int border_mode, void* stream);

/* ---------------------------------------------------------------------------------------------------
 * Upsample(f) block.  replaces: network/MaskFlownet.py:35-62 (edge pad + fixed-kernel Deconvolution +
 * crop), used stand-alone at pipeline.py:31-32,137-138 and MaskFlownet.py:308,311 and inside the loss.
 *   out[f*i+r] = in[i]*(1-r/f) + in[min(i+1,H-1)]*(r/f), separable.  in (planes,H,W) -> out (planes,fH,fW)
 * scale multiplies the result (Upsample(4)(flow2)*self.scale, MaskFlownet.py:311).
 * ------------------------------------------------------------------------------------------------- */
MFN_API int mfn_upsample_forward(const float* in, float* out, int planes, int H, int W, int factor,
                         float scale, void* stream);
/* grad_in (planes,H,W) = transposed operator applied to grad_out (planes,fH,fW), times scale. */
MFN_API int mfn_upsample_backward(const float* grad_out, float* grad_in, int planes, int H, int W, int factor,
                          float scale, void* stream);

/* ---------------------------------------------------------------------------------------------------
 * Image warp (signature-faithful pieces).
 * replaces: F.GridGenerator(data=flow_xy, transform_type='warp') -- network/layer.py:17,29
 *           F.BilinearSampler(data, grid)                        -- network/layer.py:18,30
 * grid[:,0] = (flow[:,0]+x)/((W-1)/2) - 1, grid[:,1] = (flow[:,1]+y)/((H-1)/2) - 1; the sampler maps
 * back with x=(gx+1)(W-1)/2 and reads the four neighbours, each only when inside the image.
 * ------------------------------------------------------------------------------------------------- */
MFN_API int mfn_grid_generator_warp_forward(const float* flow_xy, float* grid, int N, int H, int W,
                                    void* stream);
MFN_API int mfn_bilinear_sampler_forward(const float* data, const float* grid, float* out, int N, int C,
                                 int H, int W, int OH, int OW, void* stream);

/* GridGenerator('warp') backward: grad_flow (N,2,H,W) overwritten,
 * channel 0 = grad_grid[:,0] * 2/(W-1), channel 1 = grad_grid[:,1] * 2/(H-1). */
MFN_API int mfn_grid_generator_warp_backward(const float* grad_grid, float* grad_flow, int N, int H, int W,
                                             void* stream);

/* BilinearSampler backward (MXNet BilinearSamplerBackward; equal to torch grid_sample(bilinear, zeros,
 * align_corners=True) backward).  grad_out (N,C,OH,OW); data, grid as in the forward.
 *   grad_data (N,C,H,W) ACCUMULATED (caller zero-fills, atomics) or NULL;
 *   grad_grid (N,2,OH,OW) overwritten (no atomics, bit-reproducible) or NULL.
 * A corner outside the image reads 0 and receives no data gradient; at integer sample positions the position
 * derivative is the one from the floor side. */
MFN_API int mfn_bilinear_sampler_backward(const float* grad_out, const float* data, const float* grid,
                                          float* grad_data, float* grad_grid, int N, int C, int H, int W, int OH,
                                          int OW, void* stream);

/* Fused cascade-input builder.  replaces: network/MaskFlownet.py:308-313
 *     mask0 = sigmoid(Upsample(4)(mask2)) - 0.5
 *     c40   = concat( warp(im2, Upsample(4)(flow2)*scale), mask0 )       [layer.py:8-18]
 *     c30   = concat( im1, zeros_like(mask0) )
 *   im1, im2 (N,Ci,H,W); flow_q (N,2,H/4,W/4) (y,x); mask_q (N,1,H/4,W/4)
 *   c30, c40 (N,Ci+1,H,W); c30 may be NULL (then only c40 is produced). */
MFN_API int mfn_image_warp_concat_forward(const float* im1, const float* im2, const float* flow_q,
                                  const float* mask_q, float* c30, float* c40, int N, int Ci, int H,
                                  int W, float flow_scale, void* stream);

/* Backward of mfn_image_warp_concat_forward with respect to c40 (grad_c40 (N,Ci+1,H,W); the gradient of c30 with
 * respect to im1 is its first Ci channels).
 *   grad_flow_up (N,2,H,W) (y,x), overwritten or NULL: gradient w.r.t. Upsample(4)(flow_q), flow_scale included;
 *   grad_mask_up (N,1,H,W), overwritten or NULL: grad_c40[:,Ci] * sigmoid'(Upsample(4)(mask_q));
 *   grad_im2 (N,Ci,H,W) ACCUMULATED (caller zero-fills, atomics) or NULL.
 * grad_flow_up and grad_mask_up use no atomics (bit-reproducible).  The transposed Upsample(4) to (N,2|1,H/4,W/4) is
 * mfn_upsample_backward, as for mfn_warp_mask_backward. */
MFN_API int mfn_image_warp_concat_backward(const float* grad_c40, const float* im2, const float* flow_q,
                                           const float* mask_q, float* grad_im2, float* grad_flow_up,
                                           float* grad_mask_up, int N, int Ci, int H, int W, float flow_scale,
                                           void* stream);

/* ---------------------------------------------------------------------------------------------------
 * Decoder dense-block convolution (SURVEY.md section 8f, row N2).
 * replaces: the `conv` blocks of the decoder / context network, nn.Conv2D(3x3, stride 1, pad 1) + LeakyReLU(0.1)
 *           (network/MaskFlownet.py:166-175) together with the concat that follows each of them,
 *           x = F.concat(convL_i(x), x)  (:219-223, 237-241, 255-259, 273-277, 291-295).
 * The input channels are read IN PLACE from a wider NCHW buffer (x_batch_stride = elements between samples) and the
 * bias + LeakyReLU'ed output channels are written into another slice of (possibly the same) buffer, so the dense block
 * needs no concat copies.  fp32-accurate tensor-core arithmetic (bf16 hi/lo split, 3 MMAs per product, fp32 accumulate).
 * Weights are packed once per layer: mfn_conv3x3_packed_bytes() -> caller allocates -> mfn_conv3x3_pack_weights().
 * Cout <= 256.  leaky_slope = 1 disables the activation.
 * Two kernels serve it: warpgroup MMAs (csrc/conv3x3_wgmma.cu, default; tuning key "conv_wgmma") and
 * the mma.sync kernel (csrc/conv3x3.cu, stride 1, Cout <= 128); the packed buffer holds both weight images.
 * mfn_conv3x3_forward_ex adds
 *   - stride 2 (pad 1, dilation 1) = the feature pyramid's down-sampling convolutions conv{L}a / conv{L}x
 *     (network/MaskFlownet.py:147-165, 200-201: nn.Conv2D(3x3, strides=2, padding=1) + LeakyReLU); H, W are the INPUT
 *     extents, the output is ((H-1)/stride+1, (W-1)/stride+1);
 *   - out_mode MFN_CONV_OUT_DEPTH_TO_SPACE2: conv channel (2 py + px) * F + f is written to out[n][f][2y+py][2x+px]
 *     (F = Cout / 4, bias has F entries, out is (N, F, 2H, 2W)).  With the weight re-arrangement of INTEGRATION.md this
 *     is the decoder's nn.Conv2DTranspose(kernel 4, stride 2, pad 1) `upfeat` layers (network/MaskFlownet.py:225, 243 ...).
 * ------------------------------------------------------------------------------------------------- */
MFN_API long long mfn_conv3x3_packed_bytes(int Cin, int Cout);
MFN_API int mfn_conv3x3_pack_weights(const float* weight /* (Cout,Cin,3,3) */, void* packed, int Cin, int Cout,
                                     void* stream);
MFN_API int mfn_conv3x3_forward(const float* x, long long x_batch_stride, const void* packed_weight, const float* bias,
                                float* out, long long out_batch_stride, int N, int Cin, int H, int W, int Cout,
                                int dilation /* = padding; 1 for the decoder, 2..16 in the context network */,
                                float leaky_slope, void* stream);
#define MFN_CONV_OUT_NCHW 0
#define MFN_CONV_OUT_DEPTH_TO_SPACE2 1
/* out_mode | (k << 8), NCHW only: the first k output channels are written without the activation (a linear head that shares
 * the input pass of an activated layer; network.py folds pred_flow / pred_mask over the dense block's input into conv{L}_4) */
#define MFN_CONV_OUT_LINEAR_PREFIX(k) ((k) << 8)
MFN_API int mfn_conv3x3_forward_ex(const float* x, long long x_batch_stride, const void* packed_weight, const float* bias,
                                   float* out, long long out_batch_stride, int N, int Cin, int H, int W, int Cout,
                                   int stride, int dilation, int out_mode, float leaky_slope, void* stream);
/* mfn_conv3x3_forward_ws = mfn_conv3x3_forward_ex that may borrow a caller-owned fp32 scratch buffer: layers on the small
 * pyramid levels (levels 5-6 of network/MaskFlownet.py: fewer output tiles than SMs, up to 43 input-channel chunks walked
 * serially per tile) are then split over the input channels -- k CTAs per tile write partial sums to the workspace, a second
 * launch adds them, the bias and the activation.  mfn_conv3x3_workspace_bytes returns the bytes that plan needs (0: the
 * layer is not split; passing a smaller or null workspace simply runs the unsplit kernel).  Results differ from the
 * unsplit kernel only by fp32 summation order. */
MFN_API long long mfn_conv3x3_workspace_bytes(int N, int Cin, int H, int W, int Cout, int stride, int dilation);
MFN_API int mfn_conv3x3_forward_ws(const float* x, long long x_batch_stride, const void* packed_weight, const float* bias,
                                   float* out, long long out_batch_stride, int N, int Cin, int H, int W, int Cout,
                                   int stride, int dilation, int out_mode, float leaky_slope, void* workspace,
                                   long long workspace_bytes, void* stream);

/* ---------------------------------------------------------------------------------------------------
 * The step either side of the network (SURVEY.md section 8f, row N3).
 * mfn_preprocess_forward replaces PipelineFlownet.predict / do_batch_mx -- network/pipeline.py:206-212 (`/ 255.0`),
 *   :85-87 (centralize: subtract the per-sample RGB mean taken over BOTH images), :122-130 (BilinearResize2D to the next
 *   multiple of 64, or to `resize`).  img1 / img2: (N,C,H,W) uint8 (is_uint8 = 1, values / 255) or float32 already in
 *   [0,1]; out1 / out2: (N,C,OH,OW) float32; rgb_mean: (N*C) float32 (the subtracted means).  OH == H and OW == W skips
 *   the resampling, like the reference.
 * mfn_postprocess_forward replaces do_batch / predict -- network/pipeline.py:137-141 (Upsample(4) of the finest
 *   prediction, BilinearResize2D back to the input size times (H/H', W/W') per flow channel) and :217-218 (NCHW -> NHWC,
 *   flip (y,x) -> (x,y)): pred (N,channels,Hq,Wq) -> out (N,H,W,channels), channels reversed when flip_channels;
 *   is_flow = 1 applies the per-channel rescale (channel 0 = y).  is_flow = 0 serves the occlusion mask (:138,142).
 * ------------------------------------------------------------------------------------------------- */
MFN_API int mfn_preprocess_forward(const void* img1, const void* img2, int is_uint8, float* out1, float* out2,
                                   float* rgb_mean, int N, int C, int H, int W, int OH, int OW, void* stream);
MFN_API int mfn_postprocess_forward(const float* pred, float* out, int N, int channels, int Hq, int Wq, int H, int W,
                                    int flip_channels, int is_flow, void* stream);

/* ---------------------------------------------------------------------------------------------------
 * Middlebury colour coding of a flow (Baker et al.; flow_vis.flow_to_color, which predict_new_data.py writes).
 *   flow_xy (N,H,W,2) float32, (x,y) = (u,v) in pixels: the layout mfn_postprocess_forward writes; 8-byte aligned.
 *   rgb (N,H,W,3) uint8 out, channels R,G,B (B,G,R when bgr).
 *   max_radius <= 0: each sample is divided by (r + 1e-5), r = its largest sqrt(u^2+v^2) (the reference's behaviour);
 *   max_radius > 0: every sample is divided by max_radius (colours comparable across the frames of a video).
 *   rad_max (N) float32 out: the radius each sample was normalised by (r, or max_radius).
 * Per pixel: rad = |(u,v)|, angle atan2(-v,-u)/pi -> blend of two neighbouring entries of a 55-entry colour wheel;
 * rad <= 1 whitens towards the centre (1 - rad (1 - col)), rad > 1 darkens (0.75 col); out = floor(255 col).
 * Any input, NaN and inf included, stays inside the wheel (such pixels get unspecified colours).  Capture-safe, no
 * allocation: a cudaMemsetAsync and a max pass (per-sample mode only), then one colouring pass.
 * ------------------------------------------------------------------------------------------------- */
MFN_API int mfn_flow_to_color(const float* flow_xy, unsigned char* rgb, float* rad_max, int N, int H, int W,
                              float max_radius, int bgr, void* stream);

/* ---------------------------------------------------------------------------------------------------
 * Deterministic mode: bit-reproducible variants of the entry points whose default kernels accumulate with fp32 atomics
 * (the scatter of a bilinear sample's gradient to its four corners, per-CTA weight partials, per-slice plane sums).  Same
 * arguments and results as the counterpart named without _det, plus a caller-owned workspace `det_ws` of `det_ws_bytes`
 * bytes (16-byte aligned; contents need not be initialised); a null or too small workspace returns MFN_ERR_INVALID_ARG.
 * Two calls with the same inputs give bit-identical outputs, whatever the GPU and the thread schedule.
 *   - Scatters (grad_x, grad_data, grad_im2) accumulate in 64-bit fixed point with integer atomics; the scale
 *     2^s is chosen on the device from a bound on the largest contribution and the largest fan-in, so no sum can overflow.
 *     Each element differs from the exact sum of its fp32 contributions by at most n * 2^-(s+1) (n = contributions to it)
 *     plus the final fp32 rounding: far below fp32 atomics' reordering noise.  NaN / inf in the bound give NaN in the output.
 *   - grad_weight of the K4 entries: per-CTA partials (128 pixels per CTA) reduced in CTA order.
 *   - mfn_preprocess_forward_det: 64 slices per plane whatever the GPU, partial sums added in slice order.
 * Workspace bytes (the formulas of maskflownet_b200/ops.py, det_workspace_bytes):
 *   mfn_warp_mask_backward_det, mfn_deformable_conv_backward_det:
 *       256 + 8*N*C*H*W + 4*F*C*9*ceil(N*H*W / 128)
 *   mfn_bilinear_sampler_backward_det:   256 + 8*N*C*H*W      (data extents)
 *   mfn_image_warp_concat_backward_det:  256 + 8*N*Ci*H*W
 *   mfn_preprocess_forward_det:          256 + 4*N*C*64
 * ------------------------------------------------------------------------------------------------- */
MFN_API int mfn_warp_mask_backward_det(const float* grad_out, const float* out, const float* conv_out,
                                       const float* x, const float* flow_up, const float* mask_up,
                                       const float* weight, float* grad_x, float* grad_flow_up,
                                       float* grad_mask_up, float* grad_weight, float* grad_bias,
                                       float* grad_tradeoff, float* grad_conv_ws, int N, int C, int H, int W,
                                       int F, float flow_scale, float level_stride, float leaky_slope,
                                       int border_mode, void* det_ws, long long det_ws_bytes, void* stream);
MFN_API int mfn_deformable_conv_backward_det(const float* grad_out, const float* data, const float* offset,
                                             const float* weight, float* grad_data, float* grad_offset,
                                             float* grad_weight, float* grad_bias, int N, int C, int H, int W,
                                             int F, int border_mode, void* det_ws, long long det_ws_bytes,
                                             void* stream);
MFN_API int mfn_bilinear_sampler_backward_det(const float* grad_out, const float* data, const float* grid,
                                              float* grad_data, float* grad_grid, int N, int C, int H, int W,
                                              int OH, int OW, void* det_ws, long long det_ws_bytes, void* stream);
MFN_API int mfn_image_warp_concat_backward_det(const float* grad_c40, const float* im2, const float* flow_q,
                                               const float* mask_q, float* grad_im2, float* grad_flow_up,
                                               float* grad_mask_up, int N, int Ci, int H, int W, float flow_scale,
                                               void* det_ws, long long det_ws_bytes, void* stream);
MFN_API int mfn_preprocess_forward_det(const void* img1, const void* img2, int is_uint8, float* out1, float* out2,
                                       float* rgb_mean, int N, int C, int H, int W, int OH, int OW, void* det_ws,
                                       long long det_ws_bytes, void* stream);

/* ---------------------------------------------------------------------------------------------------
 * GPU-side training augmentation (SURVEY.md section 8f, row N4): /root/reference/augmentation.py:168-339, constructed in
 * main.py:386-419, applied in network/pipeline.py:100-102 (`/ 255`, geo_aug, color_aug).  The random draws and the small
 * per-sample matrices derived from them are host logic (maskflownet_b200/augment.py); the kernels take the result as a
 * parameter block and are deterministic.
 *
 * mfn_geometry_augment_forward replaces GeometryAugmentation.hybrid_forward (augmentation.py:278-339) in ONE launch.
 *   img1 / img2 (N,3,H,W) and mask (N,1,H,W), or (N,1,1,1) when mask_broadcast (train_batch's default mask, pipeline.py:93-94):
 *   uint8 when is_uint8 (read as value / 255, pipeline.py:100) else float32; flow (N,2,H,W) float32, channel 0 = x.
 *   params (N,22) float32 per sample:
 *     [0:6]   affine_params  (:291-293)            the first image's 2x3 affine map, row-major, in normalised coordinates
 *     [6:12]  affine_2       (:305)                = affine_params . relative transform
 *     [12:14] rel_translation (:302), zeros when the block has none: added to the second grid (:323-324) and, times
 *             ((W-1)/2, (H-1)/2), subtracted from the flow (:303-307)
 *     [14:18] inverse_2      (:326) 2x2 applied to the sampled flow    [18:22] factor (:337) 2x2 applied to the identity grid
 *   outputs on the (TH,TW) target grid: out_img1 / out_img2 (N,3,TH,TW), out_flow (N,2,TH,TW), out_mask (N,1,TH,TW).
 *   GridGenerator('affine') and BilinearSampler semantics: MXNet's (grid x = -1 + j*2/(TW-1); zero weight for taps outside).
 * mfn_color_augment_forward replaces ColorAugmentation.hybrid_forward (augmentation.py:182-227) for both images in two
 *   launches.  img1 / img2 / out1 / out2 (N,3,H,W) float32; params (N,26) per sample:
 *     [0:9] sh_matrix (:198-200)  [9:12] contrast * channel (:218)  [12:15] channel  [15] brightness (:221)
 *     [16] exp(gamma) (:224; used when has_gamma)  [17:26] spin_matrix (:206-208), the identity without eigen_aug.
 *   noise1 / noise2: (N,3,H,W) standard-normal tensors (the reference's F.random.normal, :214), or both null: then, when
 *   noise_sigma != 0, the kernels generate the noise themselves (Philox4x32-10 keyed by `seed`, counter = pixel index).
 *   workspace: mfn_color_augment_workspace_bytes(N) bytes of caller-owned scratch (per-slice partial sums; no atomics,
 *   so the result is bit-reproducible).
 * ------------------------------------------------------------------------------------------------- */
MFN_API int mfn_geometry_augment_forward(const void* img1, const void* img2, int is_uint8, const float* flow, const void* mask,
                                         int mask_broadcast, const float* params, float* out_img1, float* out_img2,
                                         float* out_flow, float* out_mask, int N, int H, int W, int TH, int TW, void* stream);
MFN_API long long mfn_color_augment_workspace_bytes(int N);
MFN_API int mfn_color_augment_forward(const float* img1, const float* img2, const float* params, const float* noise1,
                                      const float* noise2, float noise_sigma, long long seed, float* out1, float* out2,
                                      void* workspace, long long workspace_bytes, int N, int H, int W, int has_gamma,
                                      void* stream);

/* ---------------------------------------------------------------------------------------------------
 * MultiscaleEpe('upsampling'), fused (SURVEY.md section 8f, row N2): network/MaskFlownet.py:563-611, built in
 * network/pipeline.py:39-45 (scales 64,32,16,8,4; weights .005,.01,.02,.08,.32), applied in pipeline.py:81-83,107.
 *   loss[n] = sum_s weights[s] * sum_hw( e_s * mask ) / sum_hw( mask ),
 *   e_s = sqrt( sum_c (Upsample(scales[s])(preds[s])_c - flow_c)^2 + eps )   or, q >= 0:  ( sum_c |.| + eps )^q   (q < 0: L2)
 * flow (N,2,H,W) label, mask (N,1,H,W), preds[s] (N,2,H/scales[s],W/scales[s]): device pointers; preds / grad_preds / scales /
 * weights are HOST arrays of num_scales (<= 8) entries.  forward: loss (N), mask_sum (N) (kept for backward), workspace of
 * mfn_multiscale_epe_workspace_bytes(N) bytes; one pass over flow and mask, no up-sampled tensor is materialised.
 * backward: grad_preds[s] (N,2,H/s,W/s) = d( sum_n grad_loss[n] * loss[n] ) / d preds[s], one launch, gather form, no atomics.
 * ------------------------------------------------------------------------------------------------- */
MFN_API long long mfn_multiscale_epe_workspace_bytes(int N);
MFN_API int mfn_multiscale_epe_forward(const float* flow, const float* mask, const float* const* preds, const int* scales,
                                       const float* weights, int num_scales, float eps, float q, float* loss, float* mask_sum,
                                       void* workspace, long long workspace_bytes, int N, int H, int W, void* stream);
MFN_API int mfn_multiscale_epe_backward(const float* flow, const float* mask, const float* const* preds, const int* scales,
                                        const float* weights, int num_scales, float eps, float q, const float* grad_loss,
                                        const float* mask_sum, float* const* grad_preds, int N, int H, int W, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* MASKFLOW_B200_H_ */
