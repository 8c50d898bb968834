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
/* Process-wide tuning / test knobs.  The defaults are what the library runs; tests set the others to reach a fallback at
 * small shapes, or to show that two paths give identical results.  This list is complete: any other key returns
 * MFN_ERR_INVALID_ARG.
 *   "corr_grid_cap"  default 0: > 0 caps the persistent grid of the tensor-core correlation kernels at that many CTAs
 *                    (long per-CTA tile runs)
 *   "corr_tma"       default 1: 0 = C <= 32 correlations skip the TMA pipeline kernel and take the strip-marching (ring)
 *                    kernel, which otherwise serves only the shapes the TMA kernel declines
 *   "corr_rb"        default 1: C > 32 correlations with N*H*W <= 1024 run on the row-block kernel; 2 = the row-block
 *                    kernel for every shape it fits; 0 = never (the chunked tile kernel instead)
 *   "warp_lin"       default 1: 0 = mfn_warp_mask_forward_resample takes the border-list path instead of the evaluation
 *                    through linearity
 *   "conv_wgmma"     default 1: 0 = the 3x3 convolutions the mma.sync kernel covers (stride 1, Cout <= 128, NCHW output)
 *                    run on it instead of the wgmma kernel
 *   "conv_grid_cap"  default 0: > 0 caps the persistent wgmma convolution's grid at that many CTAs (0 = one per SM)
 *   "conv_splitk"    default 1: the plan splits the input channels of small layers (<= 8 parts); 0 = never split;
 *                    k > 1 = at most k parts
 *   "conv_narrow"    default 1: 0 = every wgmma convolution takes 128-pixel tile rows (no 64-pixel rows)
 *   "conv_tma_in"    default 1: 0 = fp32 wgmma inputs are loaded per thread instead of staged by TMA
 *   "conv_dbg"       default 0: profiling switches of the wgmma convolution (2 = producers skip global loads, 4 = no
 *                    epilogue stores, 8 = no MMAs, 16 = no input path, 32 = no weight copies); any non-zero value
 *                    makes results invalid */
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
 * Two kernels serve it: warpgroup MMAs (csrc/conv3x3_wgmma.cu, default) and the mma.sync kernel (csrc/conv3x3.cu,
 * stride 1, Cout <= 128), which runs the shapes the wgmma kernel declines and everything it covers when tuning key
 * "conv_wgmma" = 0; the packed buffer holds both weight images.
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
/* out_mode | MFN_CONV_BF16 (mfn_conv3x3_forward_ex, _ws, _split): opt-in bf16 inference arithmetic.  The input and the
 * weights are each rounded once to bf16 (nearest even: the "hi" of the split), each product is the one MMA hi*hi, exact
 * in fp32, and products accumulate in fp32; bias, activation, linear prefix, depth-to-space and split-K are unchanged.
 * Each product errs by up to about 2^-7 relative (two roundings to 8 significant bits) instead of about 2^-17.  Only the wgmma kernel has this variant: the bit
 * returns MFN_ERR_UNSUPPORTED where the mma.sync kernel would run (a shape the wgmma kernel declines, or tuning "conv_wgmma" = 0).
 * mfn_conv3x3_workspace_bytes does not depend on it. */
#define MFN_CONV_BF16 0x10
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

/* Split activations (csrc/split_act.cuh): an activation of C channels stored as (N, 2, Cg, H, W, 8) bf16, Cg =
 * ceil(C/16)*2 groups of 8 channels -- per sample the bf16 "hi" image of every group, then the "lo" image of the
 * remainders (the operand split every tensor-core contraction here uses) -- 4 bytes per channel-pixel like fp32, with the
 * channels past C zero.  Stored so, a value is converted once, when written, instead of by every convolution that reads
 * it (the dense block makes each layer read everything written before it), and a convolution loads its input tiles with
 * plain tensor copies.
 * mfn_split_pack: channels [0, C) of an fp32 NCHW tensor (src_batch_stride elements between samples, 0 = C*H*W) into
 *   channels [dst_c0, dst_c0 + C) of a split buffer of dst_channels channels; the slice starts at a multiple of 16 and
 *   ends at one or at the buffer's last channel (whose pad up to the next multiple of 16 is then written as zeros).
 * mfn_conv3x3_forward_split = mfn_conv3x3_forward_ws, stride 1, reading channels [x_c0, x_c0 + Cin) of the split buffer x
 *   of x_channels channels (a slice that starts at a multiple of 16 and ends at one or at the last channel).  out_split == NULL: fp32 output to `out` as in mfn_conv3x3_forward_ws
 *   (NCHW or depth-to-space).  Otherwise the output channels past the linear prefix k (out_mode = MFN_CONV_OUT_NCHW |
 *   MFN_CONV_OUT_LINEAR_PREFIX(k), k even, Cout - k a multiple of 16) go to channels out_split_c0.. (a multiple of 16) of
 *   the split buffer out_split of out_split_channels channels, and the k prefix channels to the fp32 (N, k, H, W) `out`.
 *   Dilations >= 2 must be even.  The products and their order are those of mfn_conv3x3_forward_ws on the same fp32 values:
 *   results are bit-identical. */
MFN_API int mfn_split_pack(const float* src, long long src_batch_stride, int N, int C, int H, int W, void* dst,
                           int dst_channels, int dst_c0, void* stream);
/* bf16 activations (MFN_CONV_BF16): the split layout with ONE plane, (N, 1, Cg, H, W, 8) bf16 -- the hi image alone, every
 * value rounded once to bf16, nearest even -- 2 bytes per channel-pixel, channels past C zero.
 * mfn_bf16_pack: mfn_split_pack into a bf16-activation buffer (same arguments and slice rules).
 * mfn_conv3x3_forward_split with out_mode | MFN_CONV_BF16 reads x and writes out_split as bf16 activations; its fp32
 *   outputs (`out`: NCHW, depth-to-space or the linear prefix) stay fp32. */
MFN_API int mfn_bf16_pack(const float* src, long long src_batch_stride, int N, int C, int H, int W, void* dst,
                          int dst_channels, int dst_c0, void* stream);
MFN_API int mfn_conv3x3_forward_split(const void* x, int x_channels, int x_c0, const void* packed_weight, const float* bias,
                                      float* out, long long out_batch_stride, void* out_split, int out_split_channels,
                                      int out_split_c0, int N, int Cin, int H, int W, int Cout, int dilation, int out_mode,
                                      float leaky_slope, void* workspace, long long workspace_bytes, void* stream);

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
 * Forward-backward consistency check (Sundaram, Brox and Keutzer, ECCV 2010): which pixels of each image of a pair have
 * no consistent match in the other.
 *   flow_fw, flow_bw (N,H,W,2) float32, (x,y) in pixels: the flows image 1 -> image 2 and image 2 -> image 1, in the
 *   layout mfn_postprocess_forward writes; 8-byte aligned.
 *   occ_fw, occ_bw (N,H,W) uint8 out, 1 = occluded: the pixels of image 1 (occ_fw) / image 2 (occ_bw) that fail the test.
 * Per pixel (n,y,x) of the forward direction, (u,v) = flow_fw[n,y,x], target (qx,qy) = (x+u, y+v) in float32:
 *   outside 0 <= qx <= W-1, 0 <= qy <= H-1 (NaN included) -> 1; else (bu,bv) = flow_bw sampled bilinearly at (qx,qy)
 *   (corners floor(q) and min(floor(q)+1, extent-1), weights q - floor(q)) and
 *   occ = !((u+bu)^2 + (v+bv)^2 <= rhs && rhs finite), rhs = alpha (u^2 + v^2 + bu^2 + bv^2) + beta: NaN or inf
 *   anywhere gives 1.
 * The backward direction is the same with the roles swapped.  alpha = 0.01, beta = 0.5 are the paper's constants.
 * One launch covers both directions; no atomics (deterministic), no allocation, capture-safe.  A null pointer, an extent
 * below 1, a misaligned flow, or a negative or non-finite alpha / beta returns MFN_ERR_INVALID_ARG.
 * ------------------------------------------------------------------------------------------------- */
MFN_API int mfn_flow_consistency(const float* flow_fw, const float* flow_bw, unsigned char* occ_fw, unsigned char* occ_bw,
                                 int N, int H, int W, float alpha, float beta, void* stream);

/* ---------------------------------------------------------------------------------------------------
 * Dense point tracking (Sundaram, Brox and Keutzer, ECCV 2010): tracks chained along the forward flow, stopped by the
 * forward-backward check or at motion boundaries, and reseeded on a grid where textured cells are uncovered.
 * Frames 0..T-1 of H x W; flow_fw of frame k -> k+1 and flow_bw of k+1 -> k are (H,W,2) float32 (x,y) pixels (the layout
 * mfn_postprocess_forward writes), 8-byte aligned.  The tracker holds K slots, the first M of them for the queries.  Each
 * slot holds at most one track: pos (K,2) float32 (x,y), 8-byte aligned, and a status byte per slot and frame:
 *   0 EMPTY     no track in this slot in this frame
 *   1 TRACKED   a track continued into this frame
 *   2 BORN      a track started in this frame (seed or query)
 *   3 LEFT      the track's last frame was the previous one: its target was non-finite or left the frame
 *   4 OCCLUDED  the same, ended by the forward-backward check
 *   5 BOUNDARY  the same, ended by the motion-boundary test
 * A stopped slot's position is NaN in that frame, and the slot may be seeded again from the next frame on.  Every live
 * (TRACKED or BORN) position lies inside [0,W-1] x [0,H-1].
 *
 * mfn_track_advance: frame k -> k+1 for every slot.  A slot that is not live in frame k becomes EMPTY.  A live slot at p:
 *   1. w = flow_fw sampled bilinearly at p: corners x0 = floor(px), x1 = min(x0+1, W-1), the same in y, weights
 *      p - floor(p) (mfn_flow_consistency's rule).
 *   2. q = p + w in float32.  Non-finite or outside [0,W-1] x [0,H-1]: LEFT.
 *   3. b = flow_bw sampled at q with the same rule.  OCCLUDED unless |w+b|^2 <= alpha (|w|^2 + |b|^2) + beta with that
 *      right-hand side finite.
 *   4. At the pixel nearest p (rint, ties to even, clamped to the frame), central differences of flow_fw with the
 *      neighbours clamped to the frame, divided by their index distance (0 where the extent is 1); g = the sum of their
 *      four squares.  BOUNDARY unless g <= alpha_b |w|^2 + beta_b.
 *   5. Otherwise TRACKED at q.
 *   The first test that fires wins.  Then `cells` (Gy,Gx) uint8 is zeroed and each TRACKED slot sets the cell
 *   (floor(qx) / h, floor(qy) / h) if it lies inside the grid.  alpha = 0.01, beta = 0.5 as mfn_flow_consistency;
 *   alpha_b = 0.01, beta_b = 0.002 the paper's motion-boundary constants.
 * Grid: spacing h >= 1, Gx = W / h, Gy = H / h cells (integer division); cell (i,j) covers [ih,(i+1)h) x [jh,(j+1)h) and
 *   its seed point is (ih + h/2, jh + h/2), h/2 in integers.
 * mfn_track_texture: for each of F frames (F,H,W,3) uint8 and each seed point, lambda2 (F,Gy,Gx) float64, the smaller
 *   eigenvalue of the structure tensor: grey I = R+G+B (any channel order), gx = I(x+1,y) - I(x-1,y), gy likewise,
 *   coordinates clamped to the frame; (a,b,c) = the sums of (gx^2, gx gy, gy^2) over the 5x5 window around the seed point
 *   (window coordinates clamped), exact in int32; lambda2 = max(0, (a+c)/2 - sqrt(((a-c)/2)^2 + b^2)) in float64, every
 *   intermediate exact and the square root correctly rounded, so the value is reproducible bit for bit anywhere.
 *   lambda_max (F) float64: each frame's largest lambda2 (0 without seed points).
 * mfn_track_seed: the births of the frame f = *frame, after its advance (or after a reset, for frame 0); then *frame = f+1.
 *   - Query births: queries (M,3) float32 rows (t, x, y).  Query i with t == f is BORN at (x,y) in slot i if (x,y) lies
 *     inside [0,W-1] x [0,H-1] (and covers its cell like a TRACKED slot); otherwise LEFT, with a NaN position.
 *   - Covered cells: `cells` as the advance left it, plus the query births.
 *   - Candidates: the uncovered cells with lambda2 > 0 and lambda2 >= tau lambda_max (the product in float64 from the
 *     float32 tau).  A flat frame seeds nothing.
 *   - Assignment: the n-th candidate in row-major cell order is BORN at its seed point in the n-th free slot in slot order;
 *     the free slots are the slots M..K-1 that are EMPTY after the advance.  *dropped = the candidates left without a slot.
 *   - out_pos (K,2), out_status (K), optional (both null or neither): a copy of the frame's state.
 *   ws: caller-owned, mfn_track_seed_workspace_bytes(K) = 4 K bytes, 4-byte aligned.
 * A video starts from pos = NaN, status = EMPTY, *frame = 0: mfn_track_texture of frame 0 and mfn_track_seed.  Each next
 * frame is mfn_track_advance and mfn_track_seed; mfn_track_texture may cover many frames in one call.  No float atomics
 * (deterministic), no allocation, no host synchronisation, launch configurations depend on the extents only: a sequence
 * of calls is capture-safe and replayable.  A null pointer, an extent below 1, spacing below 1, a negative or non-finite
 * constant, a misaligned pointer, M outside [0,K] or a short workspace returns MFN_ERR_INVALID_ARG; H*W >= 2^31 or
 * F > 65535 returns MFN_ERR_ALIGNMENT.
 * ------------------------------------------------------------------------------------------------- */
MFN_API int mfn_track_texture(const unsigned char* frames, double* lambda2, double* lambda_max, int F, int H, int W,
                              int spacing, void* stream);
MFN_API int mfn_track_advance(const float* flow_fw, const float* flow_bw, float* pos, unsigned char* status,
                              unsigned char* cells, int K, int H, int W, int spacing, float alpha, float beta, float alpha_b,
                              float beta_b, void* stream);
MFN_API long long mfn_track_seed_workspace_bytes(int K);
MFN_API int mfn_track_seed(const double* lambda2, const double* lambda_max, const float* queries, int M, float* pos,
                           unsigned char* status, unsigned char* cells, int* frame, int* dropped, void* ws,
                           long long ws_bytes, float* out_pos, unsigned char* out_status, int K, int H, int W, int spacing,
                           float tau, void* stream);

/* ---------------------------------------------------------------------------------------------------
 * Frame interpolation from bidirectional flow: occlusion-weighted forward splatting of both images of each pair.
 *   img0, img1 (N,H,W,3) uint8 (any channel order); flow_fw (img0 -> img1), flow_bw (img1 -> img0) (N,H,W,2) float32,
 *   (x,y) pixels, 8-byte aligned; occ_fw, occ_bw (N,H,W) uint8 (mfn_flow_consistency's masks, nonzero = occluded);
 *   times_host: a HOST array of T times, each in (0,1); occ_weight in [0,1].  out (N,T,H,W,3) uint8.
 * For time t, every pixel p = (x,y) of img0 is a source with uv = flow_fw[p], target q = (fmaf(t,u,x), fmaf(t,v,y)) in
 * float32 and weight w = (1-t) (occ_fw[p] ? occ_weight : 1); every pixel of img1 likewise with flow_bw, occ_bw, target
 * fmaf(1-t, u, x) and weight t (occ_bw[p] ? occ_weight : 1) (1-t in float32).  A non-finite q, or one outside
 * [-1,W] x [-1,H], contributes nothing.  Otherwise each corner c of floor(q), floor(q)+1 inside [0,W-1] x [0,H-1] receives
 * b w I(p) in each colour sum and b w in the weight sum, b = (1-|qx-cx|)(1-|qy-cy|); corners outside are dropped.
 * Output pixel o: weight sum W_o >= 2^-20: rint(acc_c / W_o) (ties to even), clamped to [0,255]; otherwise (a hole)
 * rint((1-t) img0[o] + t img1[o]).
 * The sums are 64-bit fixed point added with integer atomics (scales 2^(61 - k) for the weight and 2^(53 - k) for the
 * colours, k = bit length of 2HW), so the result does not depend on the order of the atomics: bit-reproducible.  Per time
 * step: a cudaMemsetAsync of the workspace, a splat launch and a normalise launch; t goes by value, so the call is
 * capture-safe for any T.  ws: caller-owned, mfn_interpolate_frames_workspace_bytes(N,H,W) = 32 N H W bytes (one step's
 * accumulators), 16-byte aligned.  A null pointer, an extent or T below 1, a time outside (0,1) or non-finite, occ_weight
 * outside [0,1], a misaligned flow or workspace, or a short workspace returns MFN_ERR_INVALID_ARG; H*W >= 2^31 or
 * N > 65535 returns MFN_ERR_ALIGNMENT.
 * ------------------------------------------------------------------------------------------------- */
MFN_API long long mfn_interpolate_frames_workspace_bytes(int N, int H, int W);
MFN_API int mfn_interpolate_frames(const unsigned char* img0, const unsigned char* img1, const float* flow_fw,
                                   const float* flow_bw, const unsigned char* occ_fw, const unsigned char* occ_bw,
                                   unsigned char* out, void* ws, long long ws_bytes, int N, int H, int W,
                                   const float* times_host, int T, float occ_weight, void* stream);

/* ---------------------------------------------------------------------------------------------------
 * Video stabilisation: the camera's motion between two frames as a robust affine fit to the flow, and a warp of uint8
 * frames by per-frame affine maps.
 *
 * mfn_affine_motion: flow (N,H,W,2) float32 (x,y) pixels (the layout mfn_postprocess_forward writes), 8-byte aligned.
 *   Pixel p = (x,y) has target q = p + flow[p] in float64; it is valid when q lies inside [0,W-1] x [0,H-1] (a non-finite
 *   component is never inside).  Coordinates are normalised for the fit: p^ = (p - c) / s, q^ = (q - c) / s with
 *   c = ((W-1)/2, (H-1)/2) and s = max(W,H)/2.  Iteration k solves the weighted least squares
 *     M = sum w phi phi^T,  b_x = sum w phi q^_x,  b_y = sum w phi q^_y,  phi = (x^, y^, 1)   (12 float64 sums)
 *   by the adjugate of the symmetric M over det(M), and maps the solution back to pixels, A = [L | c + s t - L c] for
 *   q^ = L p^ + t.  Weights: invalid pixels 0; iteration 0: 1 (plain least squares); iteration k >= 1: the Cauchy weight
 *   w = 1 / (1 + r^2 / sigma_k^2), r^2 = |A_{k-1} p - q|^2 in pixels under the previous iteration's A (all float64),
 *   sigma_k = sigma 2^max(0, 4-k) (8 sigma, 4 sigma, 2 sigma, sigma, sigma, ...).
 *   A solve is well conditioned when the total weight M[2][2] >= 3 and det(M) > 1e-9 (tr(M)/3)^3; otherwise it writes
 *   the identity, which the next iteration's weights then use.
 *   affine (N,2,3) float64, 8-byte aligned: the last iteration's A, A [x,y,1]^T ~ p + flow[p].  ok (N) uint8: 1 when the
 *   last solve was well conditioned.  residual (N,H,W) float32, optional (null: not written), 4-byte aligned:
 *   float(sqrt(r^2)) under the final A, NaN on invalid pixels.
 *   Each iteration is two launches: per-CTA float64 partials (each thread's pixels summed in a fixed order, the CTA's
 *   threads by a fixed tree; the number of CTAs per sample depends on H and W only) and one CTA per sample that adds them
 *   in a fixed order and solves.  No atomics (bit-reproducible), no allocation, no host synchronisation, a launch count
 *   fixed by `iterations`: capture-safe.  ws: caller-owned, mfn_affine_motion_workspace_bytes(N,H,W) bytes, 8-byte
 *   aligned.
 * mfn_warp_frames_affine: src, out (N,H,W,3) uint8 (any channel order); M (N,2,3) float64 ON THE DEVICE, 8-byte aligned,
 *   mapping output pixels to source positions.  Output pixel o = (x,y) of sample n, in float64:
 *     s = M [x,y,1]^T;  s clamped to [0,W-1] x [0,H-1] (fmin(fmax(s, 0), W-1): the border is replicated, NaN gives 0);
 *     x0 = floor(sx), x1 = min(x0+1, W-1), wx = sx - x0, the same in y (the corner rule of flowcheck.cuh's fb_sample);
 *     v = (1-wy) ((1-wx) I[y0,x0] + wx I[y0,x1]) + wy ((1-wx) I[y1,x0] + wx I[y1,x1]) per channel, evaluated in that order;
 *     out = rint(v) (ties to even), clamped to [0,255].
 *   No atomics, no allocation: deterministic and capture-safe.
 * A null pointer, an extent below 1, iterations below 1, a non-positive or non-finite sigma, a misaligned pointer or a
 * short workspace returns MFN_ERR_INVALID_ARG; H*W >= 2^31 or N > 65535 returns MFN_ERR_ALIGNMENT.
 * ------------------------------------------------------------------------------------------------- */
MFN_API long long mfn_affine_motion_workspace_bytes(int N, int H, int W);
MFN_API int mfn_affine_motion(const float* flow, double* affine, unsigned char* ok, float* residual, void* ws,
                              long long ws_bytes, int N, int H, int W, int iterations, float sigma, void* stream);
MFN_API int mfn_warp_frames_affine(const unsigned char* src, const double* M, unsigned char* out, int N, int H, int W,
                                   void* stream);

/* ---------------------------------------------------------------------------------------------------
 * Moving-object segmentation: the pixels that move relative to the camera, labelled into 8-connected objects.
 * Output frame n has two optional sides, each sample n of which lies on frame n:
 *   side a (the forward direction, frame n -> n+1): res_a (N,H,W) float32, mfn_affine_motion's residual of the forward
 *     flow; occ_a (N,H,W) uint8, its mfn_flow_consistency mask (nonzero = occluded); flow_a (N,H,W,2) float32 (x,y)
 *     pixels, the forward flow; affine_a (N,2,3) float64, the forward flow's fit A.  All four null, or none.
 *   side b (the backward direction, frame n -> n-1): res_b (N,H,W) float32 and occ_b (N,H,W) uint8, the same for the
 *     backward flow.  Both null, or neither.  Both sides null gives empty frames.
 * Rule, per frame and pixel p:
 *   a = res_a(p), defined when finite and occ_a(p) = 0; b likewise from side b.  s = min(a, b) when both are defined, the
 *   defined one when one is, undefined otherwise.  L = {p : s(p) >= tau_lo} in float32.  The components are the
 *   8-connected components of L; one is kept when some pixel of it has s >= tau_hi and its area is >= min_area.  Kept
 *   components are numbered 1, 2, ... in raster order of their first pixel (smallest y W + x), up to max_objects.
 *   labels (N,H,W) uint8: the component's number, 0 for the background, for components not kept and for kept ones past
 *   max_objects; count (N) int32 = min(kept, max_objects), dropped (N) int32 = max(0, kept - max_objects).
 *   objects (N,max_objects,10) float64, row j < count for label j + 1 (rows past count are 0):
 *     area, x0, y0, x1, y1 (inclusive box), cx, cy (the sums of x and of y, exact 64-bit integers, over the area),
 *     peak (the largest s), dx, dy: the mean over the object's pixels where a is defined of
 *     d = (p + flow_a(p)) - A p, each component evaluated in float64 as (x + u) - ((A00 x + A01 y) + A02) with every
 *     operation rounded on its own and clamped to [-2^16, 2^16]; NaN where a is defined nowhere in the object (always on
 *     a side-a-less frame).  The sums of d are 64-bit fixed point at scale 2^S, S = 46 - k, k the bit length of H W:
 *     |dx - mean(d)| <= 2^-(S+1) + 2^-50 (1 + |mean(d)|).
 * The union-find links the larger root under the smaller (parent[i] <= i), so a component's root is its first pixel
 * whatever order the unions run in; every sum is an integer atomic, the score and peak are exact float32: the result is
 * bit-reproducible.  11 launches whatever the content, no allocation, no host synchronisation: capture-safe.
 * ws: caller-owned, mfn_motion_segment_workspace_bytes(N,H,W) bytes, 16-byte aligned: 4 H W bytes of parents per frame,
 * 12 bytes per possible component (at most ceil(H/2) ceil(W/2) per frame) and 16 KiB per frame for the objects.
 * A null pointer (or an incomplete side), an extent below 1, a non-finite tau or tau_lo > tau_hi, min_area below 1,
 * max_objects outside [1,255], a misaligned pointer or a short workspace returns MFN_ERR_INVALID_ARG; H*W >= 2^31 or
 * N > 65535 returns MFN_ERR_ALIGNMENT.
 * ------------------------------------------------------------------------------------------------- */
MFN_API long long mfn_motion_segment_workspace_bytes(int N, int H, int W);
MFN_API int mfn_motion_segment(const float* res_a, const unsigned char* occ_a, const float* res_b,
                               const unsigned char* occ_b, const float* flow_a, const double* affine_a,
                               unsigned char* labels, double* objects, int* count, int* dropped, void* ws,
                               long long ws_bytes, int N, int H, int W, float tau_lo, float tau_hi, int min_area,
                               int max_objects, void* stream);

/* ---------------------------------------------------------------------------------------------------
 * Video denoising: each frame averaged with its neighbours aligned along chained bidirectional flow, every neighbour
 * weighted by a patch distance so that a wrong flow does not ghost (flow-guided temporal non-local means).
 *
 * mfn_denoise_frames: frames (S,H,W,3) uint8 (any channel order), a ring: frame t sits in slot t mod S.  flow_fw,
 *   flow_bw (S,H,W,2) float32 (x,y) pixels (the layout mfn_postprocess_forward writes), rings, 8-byte aligned: slot
 *   t mod S holds pair (t, t+1), flow_fw of t -> t+1 and flow_bw of t+1 -> t.  out (N,H,W,3) uint8: frames t0 .. t0+N-1.
 *   The video's frames are [t_lo, t_hi]; every window is clamped to them.  A plain clip is S = T, t_lo = 0, t_hi = T-1
 *   (its last flow slot is never read).
 *   Trajectory of pixel p of frame t, in float32, q_0 = p:
 *     forward, k = 1 .. min(R, t_hi - t): w = flow_fw[t+k-1] sampled bilinearly at q_{k-1} (corners x0 = floor(qx),
 *       x1 = min(x0+1, W-1), the same in y, weights q - floor(q): mfn_flow_consistency's rule); q = q_{k-1} + w.  The
 *       chain stops if q is non-finite or outside [0,W-1] x [0,H-1], or unless |w+b|^2 <= alpha (|w|^2 + |b|^2) + beta
 *       with that right-hand side finite, b = flow_bw[t+k-1] sampled at q (mfn_track_advance, steps 1-3).  Otherwise
 *       q_k = q and a_k(p) = frame t+k sampled bilinearly at q_k per channel with the same corner rule,
 *       fl((1-wy) fl((1-wx) A + wx B) + wy fl((1-wx) C + wx D)) in float32 (flowcheck.cuh's fb_lerp).
 *     backward, k = 1 .. min(R, t - t_lo): the same with flow_bw[t-k] as the step, flow_fw[t-k] as the check and frame
 *       t-k as the colour.
 *     Once a chain stops, a_k is undefined for that k and every later k of its direction.
 *   Weight of neighbour k at p (float32): 0 where a_k(p) is undefined; otherwise over the offsets o in [-r,r]^2 (oy
 *     outer, ox inner, ascending) for which p+o lies in the frame and a_k(p+o) is defined, n of them,
 *     D = the sum over o and the channels c = 0,1,2 of (a_k,c(p+o) - I_t,c(p+o))^2 in that order, d2 = D / (3n), and
 *     w_k = expf(-fmaxf(d2 - 2 sigma^2, 0) / (h_factor sigma)^2), with 2 sigma^2 = 2 (sigma sigma) and
 *     (h_factor sigma)^2 = hs hs, hs = h_factor sigma, each rounded to float32.
 *   Output, per channel: out = rint((I_t(p) + sum_k w_k a_k(p)) / (1 + sum_k w_k)) (ties to even), clamped to [0,255];
 *     the sums run over the forward neighbours k = 1..R, then the backward ones k = 1..R, in float32.  R = 0, or no
 *     defined neighbour, returns the input.
 *   radius R >= 0, patch r in [0, 8] (r above 8 returns MFN_ERR_UNSUPPORTED), sigma > 0 in grey levels, h_factor > 0;
 *   alpha = 0.01, beta = 0.5 are mfn_flow_consistency's constants.  The ring must hold every frame the windows read:
 *   t_lo <= t0, t0+N-1 <= t_hi and min(t_hi, t0+N-1+R) - max(t_lo, t0-R) + 1 <= S.
 *   One launch of 16 x 16-pixel tiles per frame, (16+2r)^2 x 32 bytes of shared memory per CTA.  No atomics (the result
 *   does not depend on the thread schedule or on the other frames of the call), no allocation, no host synchronisation;
 *   the launch configuration depends on the extents only: capture-safe.
 * mfn_noise_sigma: frames (F,H,W,3) uint8 -> sigma (F) float64, 8-byte aligned: Immerkaer's estimator (CVIU 1996),
 *   S = the sum over the three channels and the interior pixels (1 <= x <= W-2, 1 <= y <= H-2) of
 *   |I * [[1,-2,1],[-2,4,-2],[1,-2,1]]|, exact in int64; sigma = max(0.5, sqrt(pi/2) S / (18 (W-2) (H-2))), evaluated
 *   in float64 as (1.2533141373155003 S) / ((18 (W-2)) (H-2)).  The floor of 0.5 grey levels keeps sigma > 0 on clean
 *   or flat frames.  Bit-reproducible; one CTA per frame.  H or W below 3 returns MFN_ERR_INVALID_ARG.
 * A null pointer, an extent below 1, R or r below 0, a non-positive or non-finite sigma or h_factor, a negative or
 * non-finite alpha or beta, a window outside [t_lo, t_hi] or not held by the ring, or a misaligned flow returns
 * MFN_ERR_INVALID_ARG; H*W >= 2^31 or N (F) > 65535 returns MFN_ERR_ALIGNMENT.
 * ------------------------------------------------------------------------------------------------- */
MFN_API int mfn_denoise_frames(const unsigned char* frames, const float* flow_fw, const float* flow_bw,
                               unsigned char* out, int S, int H, int W, int t0, int N, int t_lo, int t_hi, int radius,
                               int patch, float sigma, float h_factor, float alpha, float beta, void* stream);
MFN_API int mfn_noise_sigma(const unsigned char* frames, double* sigma, int F, int H, int W, void* stream);

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

/* ---------------------------------------------------------------------------------------------------
 * Unsupervised losses on unlabelled frame pairs (UnFlow, Meister, Hur and Roth, AAAI 2018): an occlusion-masked census
 * distance between image 1 and image 2 warped by the flow, and a second-order, edge-aware flow smoothness.
 * All tensors float32 NCHW (occ uint8), device pointers, 4-byte aligned.
 *
 * Census.  img1, img2w (N,3,H,W) RGB in [0,1]; occ (N,H,W) uint8, nonzero = occluded (left out).
 *   I = 255 (0.2989 R + 0.5870 G + 0.1140 B).  Interior pixels p: 3 <= x <= W-4, 3 <= y <= H-4.  Over the 48 offsets o
 *   of {-3..3}^2 without (0,0):  t(I,p,o) = D / sqrt(0.81 + D^2), D = I(p+o) - I(p);  s = t(I1,p,o) - t(I2w,p,o);
 *   d(p) = sum_o s^2 / (0.1 + s^2);  rho(d) = (d^2 + 1e-6)^0.45;  v(p) = 1 - occ(p) on interior pixels, 0 elsewhere.
 *   forward:  loss[n] = sum_p v rho(d) / max(vsum[n], 1), vsum[n] = sum_p v (N floats each);
 *             coef (N,H,W) = v rho'(d), the per-pixel factor the backward reads;
 *             ws: 8*N*ceil(H/8)*ceil(W/32) bytes of caller-owned scratch (per-tile partial sums, added in a fixed order).
 *   backward: g_img2w (N,3,H,W) = d( sum_n g_loss[n] loss[n] ) / d img2w, every element written (a gather).  img1 gets
 *             no gradient.
 * Smoothness.  flow (N,2,H,W) (either channel order: both are summed alike), img (N,3,H,W) the image whose edges weight it.
 *   d2x F_c(p) = F_c(x-1) - 2 F_c(x) + F_c(x+1) on 1 <= x <= W-2, wx(p) = exp(-10 (1/3) sum_k |img_k(x+1) - img_k(x-1)| / 2),
 *   the same in y.  forward: loss[n] = sum_{c,p} wx |d2x F_c| / (2 H (W-2)) + sum_{c,p} wy |d2y F_c| / (2 (H-2) W)
 *   (a direction with no pixels adds 0); ws: 8*N*ceil(H*W/256) bytes.
 *   backward: g_flow (N,2,H,W) = d( sum_n g_loss[n] loss[n] ) / d flow, with d|z|/dz = sign(z) (0 at 0); a 3-tap gather
 *   per direction, every element written.  img gets no gradient.
 * Shapes below 7 (census) or 3 (smoothness) in a dimension are legal: no interior pixels, loss 0, gradient 0.  No atomics:
 * results are bit-reproducible.  A null pointer, an extent below 1, a misaligned pointer, N > 65535, 3*H*W >= 2^31 or a
 * too small workspace returns MFN_ERR_INVALID_ARG.
 * ------------------------------------------------------------------------------------------------- */
MFN_API int mfn_census_loss_forward(const float* img1, const float* img2w, const unsigned char* occ, float* coef, float* vsum,
                                    float* loss, void* ws, long long ws_bytes, int N, int H, int W, void* stream);
MFN_API int mfn_census_loss_backward(const float* img1, const float* img2w, const float* coef, const float* vsum,
                                     const float* g_loss, float* g_img2w, int N, int H, int W, void* stream);
MFN_API int mfn_smoothness_loss_forward(const float* flow, const float* img, float* loss, void* ws, long long ws_bytes, int N,
                                        int H, int W, void* stream);
MFN_API int mfn_smoothness_loss_backward(const float* flow, const float* img, const float* g_loss, float* g_flow, int N,
                                         int H, int W, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* MASKFLOW_B200_H_ */
