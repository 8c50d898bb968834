"""Tensor-level operators of the MaskFlownet hot path, backed by libmaskflow_b200.so (hand-written sm_90a CUDA).

Every function takes / returns torch CUDA float32 NCHW tensors and mirrors one MXNet operator (or one fused group of
them) used by the reference; keyword names follow the MXNet operators so that the `F` shim in maskflownet_b200.mx can
forward the reference's calls verbatim.  PyTorch is only the allocator / stream / autograd plumbing here: the arithmetic
runs in the library, on the caller's current stream, and there is no CPU or eager fallback.

Reference call sites (under /root/reference):
  correlation            network/MaskFlownet.py:193-195, 440-441
  deformable_convolution network/layer.py:117-124
  warp_mask              network/MaskFlownet.py:228-233 (and :246-251, :264-269, :282-287; cascade :463-466 ...)
  upsample               network/MaskFlownet.py:35-62
  grid_generator_warp / bilinear_sampler / reconstruction2d   network/layer.py:8-18
  image_warp_concat      network/MaskFlownet.py:308-313

Under torch.use_deterministic_algorithms(True) the ops whose default kernels accumulate with fp32 atomics (the backward of
deformable_convolution, warp_mask, bilinear_sampler and image_warp_concat, and preprocess) call the *_det entry points
instead: bit-identical results from run to run, no warning needed (see deterministic()).
"""
from __future__ import annotations

import ctypes
from typing import Optional, Tuple

import torch

from . import _lib
from ._lib import MaskflowError

CORR_AUTO, CORR_GENERIC, CORR_SIMT, CORR_MMA_BF16X3 = 0, 1, 2, 3
BORDER_MXNET15, BORDER_ZERO_CORNER = 0, 1


def _chk(t: Optional[torch.Tensor], name: str, optional: bool = False) -> Optional[torch.Tensor]:
    if t is None:
        if optional:
            return None
        raise MaskflowError(f"{name}: tensor required")
    if not t.is_cuda:
        raise MaskflowError(f"{name}: expected a CUDA tensor (got {t.device}); the hot path has no CPU implementation")
    if t.dtype != torch.float32:
        raise MaskflowError(f"{name}: expected float32, got {t.dtype}")
    return t.contiguous()


def _needs_grad(*tensors) -> bool:
    return torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in tensors)


def _no_grad_path(name: str, *tensors) -> None:
    """Forward-only kernels: refuse to silently cut the autograd graph (ADVICE r1): raise when grad mode is on and any
    operand requires grad."""
    if _needs_grad(*tensors):
        raise MaskflowError(f"{name} is forward-only (no backward kernel): call it under torch.no_grad() or detach the "
                            f"operands -- an operand requires grad")


def _p(t: Optional[torch.Tensor]):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _call(name, dev, *args):
    with torch.cuda.device(dev):
        _lib.call(name, *args, _stream())


# ----------------------------------------------------------------------------------------------------------
# Deterministic mode
# ----------------------------------------------------------------------------------------------------------
def deterministic() -> bool:
    """True under torch.use_deterministic_algorithms(True) (warn_only included): the ops whose default kernels accumulate
    with fp32 atomics then call their *_det entry points, which give bit-identical results from run to run."""
    return torch.are_deterministic_algorithms_enabled()


def det_workspace_bytes(op: str, N: int, C: int, H: int, W: int, F: int = 0) -> int:
    """Bytes of the det_ws workspace of the *_det entry points (include/maskflow_b200.h, "Deterministic mode").
    op: "warp_mask" / "deformable_conv" (x (N,C,H,W), F filters), "bilinear_sampler" (data (N,C,H,W)), "image_warp_concat"
    (im2 (N,C,H,W)), "preprocess" (images (N,C,H,W))."""
    if op in ("warp_mask", "deformable_conv"):
        return 256 + 8 * N * C * H * W + 4 * F * C * 9 * (-(-N * H * W // 128))
    if op in ("bilinear_sampler", "image_warp_concat"):
        return 256 + 8 * N * C * H * W
    if op == "preprocess":
        return 256 + 4 * N * C * 64
    raise MaskflowError(f"det_workspace_bytes: unknown op {op!r}")


def _det_ws(nbytes: int, dev):
    return torch.empty(nbytes, dtype=torch.uint8, device=dev)


# ----------------------------------------------------------------------------------------------------------
# Correlation
# ----------------------------------------------------------------------------------------------------------
def correlation_out_shape(H, W, pad_size, kernel_size, max_displacement, stride1, stride2):
    kr = (kernel_size - 1) // 2
    border = max_displacement + kr
    oh = -(-(H + 2 * pad_size - 2 * border) // stride1)
    ow = -(-(W + 2 * pad_size - 2 * border) // stride1)
    g = 2 * (max_displacement // stride2) + 1
    return g * g, oh, ow


def _correlation_forward(d1, d2, pad_size, kernel_size, max_displacement, stride1, stride2, is_multiply, leaky_slope,
                         algo, out=None):
    N, C, H, W = d1.shape
    D, OH, OW = correlation_out_shape(H, W, pad_size, kernel_size, max_displacement, stride1, stride2)
    if OH < 1 or OW < 1:
        raise MaskflowError("correlation: empty output")
    if out is None:
        out = torch.empty((N, D, OH, OW), device=d1.device, dtype=torch.float32)
        obs = 0
    else:
        # `out` may be a channel-slice view [:, :D] of a wider NCHW buffer (pre-allocated concat target)
        if out.shape != (N, D, OH, OW) or out.dtype != torch.float32 or out.device != d1.device:
            raise MaskflowError("correlation: out has the wrong shape / dtype / device")
        if out.stride()[1:] != (OH * OW, OW, 1):
            raise MaskflowError("correlation: out must be dense in (C,H,W)")
        obs = out.stride(0)
    _call("mfn_correlation_forward", d1.device, _p(d1), _p(d2), _p(out), N, C, H, W, pad_size, kernel_size,
          max_displacement, stride1, stride2, int(bool(is_multiply)), obs, float(leaky_slope), int(algo))
    return out


class _CorrelationFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, d1, d2, pad_size, kernel_size, max_displacement, stride1, stride2, is_multiply, leaky_slope, algo):
        res = _correlation_forward(d1, d2, pad_size, kernel_size, max_displacement, stride1, stride2, is_multiply,
                                   leaky_slope, algo, None)
        ctx.cfg = (pad_size, kernel_size, max_displacement, stride1, stride2, is_multiply, leaky_slope)
        ctx.save_for_backward(d1, d2, res)
        return res

    @staticmethod
    def backward(ctx, go):
        pad_size, kernel_size, md, s1, s2, mul, slope = ctx.cfg
        if not (kernel_size == 1 and s1 == 1 and s2 == 1 and mul and pad_size == md and md in (2, 4)):
            raise MaskflowError("correlation backward is implemented for the reference regime only "
                                "(kernel_size=1, strides=1, multiply, pad_size==max_displacement in {2,4})")
        d1, d2, res = ctx.saved_tensors
        N, C, H, W = d1.shape
        go = go.contiguous()
        g1 = torch.empty_like(d1) if ctx.needs_input_grad[0] else None
        g2 = torch.empty_like(d2) if ctx.needs_input_grad[1] else None
        fuse = slope != 1.0  # res was allocated dense by forward, go made dense above: identical strides
        _call("mfn_correlation_backward", d1.device, _p(go), _p(res) if fuse else None, _p(d1), _p(d2), _p(g1),
              _p(g2), N, C, H, W, md, go.stride(0), float(slope))
        return (g1, g2) + (None,) * 8


def correlation(data1, data2, pad_size=4, kernel_size=1, max_displacement=4, stride1=1, stride2=1, is_multiply=1,
                leaky_slope=1.0, algo=CORR_AUTO, out=None):
    """MXNet F.Correlation (+ optional fused LeakyReLU).  out[n,q,i,j], q=(dy+md)*(2md+1)+(dx+md)."""
    d1, d2 = _chk(data1, "correlation.data1"), _chk(data2, "correlation.data2")
    if d1.shape != d2.shape or d1.dim() != 4:
        raise MaskflowError(f"correlation: data1/data2 must be 4-D with equal shapes, got {tuple(d1.shape)} "
                            f"and {tuple(d2.shape)}")
    args = (int(pad_size), int(kernel_size), int(max_displacement), int(stride1), int(stride2), int(bool(is_multiply)),
            float(leaky_slope), int(algo))
    if out is not None:
        # writing into a caller-provided (possibly channel-sliced) buffer is an inference-only fast path
        if torch.is_grad_enabled() and (d1.requires_grad or d2.requires_grad):
            raise MaskflowError("correlation: out= cannot be combined with autograd")
        return _correlation_forward(d1, d2, *args, out)
    return _CorrelationFn.apply(d1, d2, *args)


# ----------------------------------------------------------------------------------------------------------
# Deformable convolution (signature-faithful)
# ----------------------------------------------------------------------------------------------------------
class _DeformConvFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, offset, weight, bias, border_mode):
        N, C, H, W = x.shape
        Fo = weight.shape[0]
        out = torch.empty((N, Fo, H, W), device=x.device, dtype=torch.float32)
        _call("mfn_deformable_conv_forward", x.device, _p(x), _p(offset), _p(weight), _p(bias), _p(out), N, C, H, W,
              Fo, 3, 3, 1, 1, 1, 1, 1, 1, 1, 1, int(border_mode))
        ctx.border_mode = border_mode
        ctx.has_bias = bias is not None
        ctx.save_for_backward(x, offset, weight)
        return out

    @staticmethod
    def backward(ctx, go):
        x, offset, weight = ctx.saved_tensors
        N, C, H, W = x.shape
        Fo = weight.shape[0]
        go = go.contiguous()
        need = ctx.needs_input_grad
        gx = torch.zeros_like(x) if need[0] else None
        goff = torch.empty_like(offset) if need[1] else None
        gw = torch.zeros_like(weight) if need[2] else None
        gb = torch.zeros(Fo, device=x.device, dtype=torch.float32) if (ctx.has_bias and need[3]) else None
        args = (_p(go), _p(x), _p(offset), _p(weight), _p(gx), _p(goff), _p(gw), _p(gb), N, C, H, W, Fo, int(ctx.border_mode))
        if deterministic():
            nb = det_workspace_bytes("deformable_conv", N, C, H, W, Fo)
            _call("mfn_deformable_conv_backward_det", x.device, *args, _p(_det_ws(nb, x.device)), nb)
        else:
            _call("mfn_deformable_conv_backward", x.device, *args)
        return gx, goff, gw, gb, None


def deformable_convolution(data, offset, weight, bias=None, kernel=(3, 3), stride=(1, 1), dilate=(1, 1), pad=(1, 1),
                           num_filter=None, num_group=1, num_deformable_group=1, no_bias=False, layout="NCHW",
                           border_mode=BORDER_MXNET15):
    """MXNet F.contrib.DeformableConvolution with the reference's kwargs (network/layer.py:91-95)."""
    x, off, w = _chk(data, "deformable_convolution.data"), _chk(offset, "deformable_convolution.offset"), \
        _chk(weight, "deformable_convolution.weight")
    b = None if no_bias else _chk(bias, "deformable_convolution.bias", optional=True)
    if (tuple(kernel), tuple(stride), tuple(dilate), tuple(pad), num_group, num_deformable_group, layout) != \
            ((3, 3), (1, 1), (1, 1), (1, 1), 1, 1, "NCHW"):
        raise MaskflowError("deformable_convolution: only kernel 3x3 / stride 1 / dilate 1 / pad 1 / one group / NCHW "
                            "is implemented (the reference's only configuration)")
    N, C, H, W = x.shape
    if w.shape[1:] != (C, 3, 3) or off.shape != (N, 18, H, W):
        raise MaskflowError(f"deformable_convolution: inconsistent shapes x={tuple(x.shape)} offset={tuple(off.shape)} "
                            f"weight={tuple(w.shape)}")
    if num_filter is not None and num_filter != w.shape[0]:
        raise MaskflowError("deformable_convolution: num_filter does not match weight.shape[0]")
    if b is not None and b.shape != (w.shape[0],):
        raise MaskflowError("deformable_convolution: bias shape mismatch")
    return _DeformConvFn.apply(x, off, w, b, int(border_mode))


# ----------------------------------------------------------------------------------------------------------
# Fused warp of one pyramid level
# ----------------------------------------------------------------------------------------------------------
class _WarpMaskFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, flow_c, mask_c, weight, bias, tradeoff, scale, stride, up, slope, border_mode):
        N, C, H, W = x.shape
        Fo = weight.shape[0]
        dev = x.device
        out = torch.empty((N, Fo, H, W), device=dev, dtype=torch.float32)
        flow_up = torch.empty((N, 2, H, W), device=dev, dtype=torch.float32)
        mask_up = torch.empty((N, 1, H, W), device=dev, dtype=torch.float32) if mask_c is not None else None
        training = any(ctx.needs_input_grad)
        conv_out = torch.empty_like(out) if (training and mask_c is not None) else None
        _call("mfn_warp_mask_forward", dev, _p(x), _p(flow_c), _p(mask_c), _p(weight), _p(bias), _p(tradeoff), _p(out),
              _p(flow_up), _p(mask_up), _p(conv_out), N, C, H, W, Fo, int(up), float(scale), float(stride),
              float(slope), int(border_mode))
        ctx.cfg = (scale, stride, up, slope, border_mode, bias is not None, tradeoff is not None)
        ctx.save_for_backward(x, weight, out, flow_up, mask_up, conv_out)
        if mask_up is None:
            mask_up = torch.empty(0, device=dev)
        return out, flow_up, mask_up

    @staticmethod
    def backward(ctx, g_out, g_flow_up, g_mask_up):
        scale, stride, up, slope, border_mode, has_bias, has_trade = ctx.cfg
        x, weight, out, flow_up, mask_up, conv_out = ctx.saved_tensors
        N, C, H, W = x.shape
        Fo = weight.shape[0]
        dev = x.device
        need = ctx.needs_input_grad  # x, flow_c, mask_c, weight, bias, tradeoff
        g_out = g_out.contiguous()
        gx = torch.zeros_like(x) if need[0] else None
        gflow = torch.empty_like(flow_up) if need[1] else None
        has_mask = mask_up is not None
        gmask = torch.empty_like(mask_up) if (has_mask and need[2]) else None
        gw = torch.zeros_like(weight) if need[3] else None
        gb = torch.zeros(Fo, device=dev, dtype=torch.float32) if (has_bias and need[4]) else None
        gtrade = torch.empty_like(out) if (has_trade and need[5]) else None
        ws = torch.empty_like(out)
        args = (_p(g_out), _p(out), _p(conv_out), _p(x), _p(flow_up), _p(mask_up) if has_mask else None, _p(weight), _p(gx),
                _p(gflow), _p(gmask), _p(gw), _p(gb), _p(gtrade), _p(ws), N, C, H, W, Fo, float(scale), float(stride),
                float(slope), int(border_mode))
        if deterministic():
            nb = det_workspace_bytes("warp_mask", N, C, H, W, Fo)
            _call("mfn_warp_mask_backward_det", dev, *args, _p(_det_ws(nb, dev)), nb)
        else:
            _call("mfn_warp_mask_backward", dev, *args)
        # gradients arriving on the up-sampled flow / mask outputs join the ones through the warp, then the
        # transposed Upsample brings them to the coarse grid
        gflow_c = gmask_c = None
        if need[1]:
            total = gflow if g_flow_up is None else gflow + g_flow_up
            gflow_c = _upsample_backward(total, up, 1.0)
        if has_mask and need[2]:
            total = gmask if (g_mask_up is None or g_mask_up.numel() == 0) else gmask + g_mask_up
            gmask_c = _upsample_backward(total, up, 1.0)
        return gx, gflow_c, gmask_c, gw, gb, gtrade, None, None, None, None, None


def warp_mask(x, flow_coarse, mask_coarse, weight, bias=None, tradeoff=None, scale=20.0, stride=32.0, upsample=2,
              leaky_slope=0.1, border_mode=BORDER_MXNET15, packed_weight=None, resample=False):
    """Fused Upsample(up)(flow, mask) -> deformable conv (all taps offset by flow*scale/stride) -> *sigmoid(mask)
    -> + tradeoff -> LeakyReLU.   Returns (warp, flow_up, mask_up or None).
    packed_weight (ops.conv3x3_pack(weight)) selects a tensor-core path when no gradient is required: with resample=True
    the operator is evaluated through linearity (plain 3x3 convolution on wgmma + bilinear re-sampling of its output +
    tap-by-tap border frame, mfn_warp_mask_forward_resample), else the gather-then-mma.sync kernel (F <= 128)."""
    x = _chk(x, "warp_mask.x")
    fc = _chk(flow_coarse, "warp_mask.flow_coarse")
    mc = _chk(mask_coarse, "warp_mask.mask_coarse", optional=True)
    w = _chk(weight, "warp_mask.weight")
    b = _chk(bias, "warp_mask.bias", optional=True)
    t = _chk(tradeoff, "warp_mask.tradeoff", optional=True)
    N, C, H, W = x.shape
    if H % upsample or W % upsample or fc.shape != (N, 2, H // upsample, W // upsample):
        raise MaskflowError(f"warp_mask: flow_coarse {tuple(fc.shape)} does not match x {tuple(x.shape)} / {upsample}")
    if mc is not None and mc.shape != (N, 1, H // upsample, W // upsample):
        raise MaskflowError("warp_mask: mask_coarse shape mismatch")
    if w.shape[1:] != (C, 3, 3):
        raise MaskflowError("warp_mask: weight must be (F, C, 3, 3)")
    if t is not None and t.shape != (N, w.shape[0], H, W):
        raise MaskflowError("warp_mask: tradeoff shape mismatch")
    needs_grad = torch.is_grad_enabled() and any(
        z is not None and z.requires_grad for z in (x, fc, mc, w, b, t))
    if packed_weight is not None and not needs_grad and resample and w.shape[0] <= 256 and H >= 4 and W >= 4:
        Fo = w.shape[0]
        out = torch.empty((N, Fo, H, W), device=x.device, dtype=torch.float32)
        ws = torch.empty(int(_lib.lib().mfn_warp_resample_workspace_bytes(N, Fo, H, W)), device=x.device, dtype=torch.uint8)
        flow_up = torch.empty((N, 2, H, W), device=x.device, dtype=torch.float32)
        mask_up = torch.empty((N, 1, H, W), device=x.device, dtype=torch.float32) if mc is not None else None
        _call("mfn_warp_mask_forward_resample", x.device, _p(x), _p(fc), _p(mc), _p(w), _p(packed_weight), _p(b), _p(t),
              _p(ws), _p(out), _p(flow_up), _p(mask_up), N, C, H, W, Fo, int(upsample), float(scale), float(stride),
              float(leaky_slope), int(border_mode))
        return out, flow_up, mask_up
    if packed_weight is not None and not needs_grad and w.shape[0] <= 128:
        Fo = w.shape[0]
        out = torch.empty((N, Fo, H, W), device=x.device, dtype=torch.float32)
        flow_up = torch.empty((N, 2, H, W), device=x.device, dtype=torch.float32)
        mask_up = torch.empty((N, 1, H, W), device=x.device, dtype=torch.float32) if mc is not None else None
        _call("mfn_warp_mask_forward_tc", x.device, _p(x), _p(fc), _p(mc), _p(packed_weight), _p(b), _p(t), _p(out),
              _p(flow_up), _p(mask_up), None, N, C, H, W, Fo, int(upsample), float(scale), float(stride),
              float(leaky_slope), int(border_mode))
        return out, flow_up, mask_up
    out, flow_up, mask_up = _WarpMaskFn.apply(x, fc, mc, w, b, t, float(scale), float(stride), int(upsample),
                                              float(leaky_slope), int(border_mode))
    return out, flow_up, (mask_up if mc is not None else None)


# ----------------------------------------------------------------------------------------------------------
# Upsample
# ----------------------------------------------------------------------------------------------------------
def _upsample_forward(x, factor, scale):
    N, C, H, W = x.shape
    out = torch.empty((N, C, H * factor, W * factor), device=x.device, dtype=torch.float32)
    _call("mfn_upsample_forward", x.device, _p(x), _p(out), N * C, H, W, int(factor), float(scale))
    return out


def _upsample_backward(go, factor, scale):
    go = go.contiguous()
    N, C, OH, OW = go.shape
    H, W = OH // factor, OW // factor
    gi = torch.empty((N, C, H, W), device=go.device, dtype=torch.float32)
    _call("mfn_upsample_backward", go.device, _p(go), _p(gi), N * C, H, W, int(factor), float(scale))
    return gi


class _UpsampleFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, factor, scale):
        ctx.cfg = (factor, scale)
        return _upsample_forward(x, factor, scale)

    @staticmethod
    def backward(ctx, go):
        factor, scale = ctx.cfg
        return _upsample_backward(go, factor, scale), None, None


def upsample(x, factor: int, scale: float = 1.0):
    """Reference Upsample(factor) block, optionally times `scale`."""
    x = _chk(x, "upsample.x")
    if factor == 1 and scale == 1.0:
        return x
    return _UpsampleFn.apply(x, int(factor), float(scale))


# ----------------------------------------------------------------------------------------------------------
# Image warp
# ----------------------------------------------------------------------------------------------------------
def _grid_generator_warp_forward(f):
    N, _, H, W = f.shape
    grid = torch.empty_like(f)
    _call("mfn_grid_generator_warp_forward", f.device, _p(f), _p(grid), N, H, W)
    return grid


class _GridGeneratorWarpFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, f):
        return _grid_generator_warp_forward(f)

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, gg):
        gg = gg.contiguous()
        N, _, H, W = gg.shape
        gf = torch.empty_like(gg)
        _call("mfn_grid_generator_warp_backward", gg.device, _p(gg), _p(gf), N, H, W)
        return gf


def grid_generator_warp(flow_xy):
    """MXNet F.GridGenerator(data=flow, transform_type='warp'); flow channels are (x, y).  Differentiable."""
    f = _chk(flow_xy, "grid_generator_warp.flow")
    if f.dim() != 4 or f.shape[1] != 2:
        raise MaskflowError("grid_generator_warp: flow must have 2 channels")
    if _needs_grad(f):
        return _GridGeneratorWarpFn.apply(f)
    return _grid_generator_warp_forward(f)


def _bilinear_sampler_forward(d, g):
    N, C, H, W = d.shape
    OH, OW = g.shape[2:]
    out = torch.empty((N, C, OH, OW), device=d.device, dtype=torch.float32)
    _call("mfn_bilinear_sampler_forward", d.device, _p(d), _p(g), _p(out), N, C, H, W, OH, OW)
    return out


class _BilinearSamplerFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, d, g):
        ctx.save_for_backward(d, g)
        return _bilinear_sampler_forward(d, g)

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, go):
        d, g = ctx.saved_tensors
        N, C, H, W = d.shape
        OH, OW = g.shape[2:]
        go = go.contiguous()
        gd = torch.zeros_like(d) if ctx.needs_input_grad[0] else None      # accumulated by the kernel
        gg = torch.empty_like(g) if ctx.needs_input_grad[1] else None
        args = (_p(go), _p(d), _p(g), _p(gd), _p(gg), N, C, H, W, OH, OW)
        if deterministic():
            nb = det_workspace_bytes("bilinear_sampler", N, C, H, W)
            _call("mfn_bilinear_sampler_backward_det", d.device, *args, _p(_det_ws(nb, d.device)), nb)
        else:
            _call("mfn_bilinear_sampler_backward", d.device, *args)
        return gd, gg


def bilinear_sampler(data, grid):
    """MXNet F.BilinearSampler(data, grid).  Differentiable with respect to data and grid."""
    d, g = _chk(data, "bilinear_sampler.data"), _chk(grid, "bilinear_sampler.grid")
    if d.dim() != 4 or g.dim() != 4 or g.shape[0] != d.shape[0] or g.shape[1] != 2:
        raise MaskflowError("bilinear_sampler: grid must be (N,2,OH,OW)")
    if _needs_grad(d, g):
        return _BilinearSamplerFn.apply(d, g)
    return _bilinear_sampler_forward(d, g)


def reconstruction2d(x, flow_yx):
    """layer.Reconstruction2D: grid = GridGenerator(flow.flip(1)); BilinearSampler(x, grid)."""
    return bilinear_sampler(x, grid_generator_warp(flow_yx.flip(1)))


def _image_warp_concat_forward(i1, i2, fq, mq, scale, want_c30):
    N, Ci, H, W = i2.shape
    c40 = torch.empty((N, Ci + 1, H, W), device=i2.device, dtype=torch.float32)
    c30 = torch.empty_like(c40) if want_c30 else None
    _call("mfn_image_warp_concat_forward", i2.device, _p(i1) if want_c30 else None, _p(i2), _p(fq), _p(mq), _p(c30),
          _p(c40), N, Ci, H, W, float(scale))
    return c30, c40


class _ImageWarpConcatFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, i1, i2, fq, mq, scale, want_c30):
        c30, c40 = _image_warp_concat_forward(i1, i2, fq, mq, scale, want_c30)
        ctx.scale = scale
        ctx.save_for_backward(i2, fq, mq)
        if c30 is None:
            c30 = torch.empty(0, device=i2.device)
        return c30, c40

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, g30, g40):
        i2, fq, mq = ctx.saved_tensors
        N, Ci, H, W = i2.shape
        need = ctx.needs_input_grad  # im1, im2, flow_q, mask_q
        # c30 = [im1 ; 0]: im1's gradient is the first Ci channels of c30's
        gi1 = g30[:, :Ci] if (need[0] and g30 is not None and g30.numel()) else None
        gi2 = gfq = gmq = None
        if g40 is not None and (need[1] or need[2] or need[3]):
            g40 = g40.contiguous()
            gi2 = torch.zeros_like(i2) if need[1] else None                    # accumulated by the kernel
            gfu = torch.empty((N, 2, H, W), device=i2.device, dtype=torch.float32) if need[2] else None
            gmu = torch.empty((N, 1, H, W), device=i2.device, dtype=torch.float32) if need[3] else None
            args = (_p(g40), _p(i2), _p(fq), _p(mq), _p(gi2), _p(gfu), _p(gmu), N, Ci, H, W, float(ctx.scale))
            if deterministic():
                nb = det_workspace_bytes("image_warp_concat", N, Ci, H, W)
                _call("mfn_image_warp_concat_backward_det", i2.device, *args, _p(_det_ws(nb, i2.device)), nb)
            else:
                _call("mfn_image_warp_concat_backward", i2.device, *args)
            # the transposed Upsample(4) brings the up-sampled gradients to the quarter-resolution grid
            gfq = _upsample_backward(gfu, 4, 1.0) if need[2] else None
            gmq = _upsample_backward(gmu, 4, 1.0) if need[3] else None
        return gi1, gi2, gfq, gmq, None, None


def image_warp_concat(im1, im2, flow_q, mask_q, scale=20.0, want_c30=True):
    """Fused cascade-input builder (network/MaskFlownet.py:308-313).  Returns (c30 or None, c40).  Differentiable with
    respect to im1 (through c30), im2, flow_q and mask_q; without a gradient to compute it is the single forward launch."""
    i2 = _chk(im2, "image_warp_concat.im2")
    i1 = _chk(im1, "image_warp_concat.im1", optional=not want_c30)
    fq, mq = _chk(flow_q, "image_warp_concat.flow_q"), _chk(mask_q, "image_warp_concat.mask_q")
    N, Ci, H, W = i2.shape
    if fq.shape != (N, 2, H // 4, W // 4) or mq.shape != (N, 1, H // 4, W // 4) or H % 4 or W % 4:
        raise MaskflowError("image_warp_concat: flow_q/mask_q must be (N,2|1,H/4,W/4)")
    if _needs_grad(i1 if want_c30 else None, i2, fq, mq):
        c30, c40 = _ImageWarpConcatFn.apply(i1 if want_c30 else None, i2, fq, mq, float(scale), bool(want_c30))
        return (c30 if want_c30 else None), c40
    return _image_warp_concat_forward(i1, i2, fq, mq, scale, want_c30)


# ----------------------------------------------------------------------------------------------------------
# Decoder dense-block convolution (in-place concat)
# ----------------------------------------------------------------------------------------------------------
def conv3x3_pack(weight: torch.Tensor) -> torch.Tensor:
    """Pack a (Cout, Cin, 3, 3) fp32 weight into the split-bf16 tile image mfn_conv3x3_forward streams."""
    w = _chk(weight.detach(), "conv3x3_pack.weight")
    Cout, Cin, kh, kw = w.shape
    if (kh, kw) != (3, 3):
        raise MaskflowError("conv3x3_pack: weight must be (Cout, Cin, 3, 3)")
    nbytes = int(_lib.lib().mfn_conv3x3_packed_bytes(Cin, Cout))
    packed = torch.empty(nbytes, dtype=torch.uint8, device=w.device)
    _call("mfn_conv3x3_pack_weights", w.device, _p(w), _p(packed), Cin, Cout)
    return packed


MFN_CONV_BF16 = 0x10   # include/maskflow_b200.h


def _out_mode(depth_to_space: bool, linear_prefix: int, bf16: bool) -> int:
    return (1 if depth_to_space else 0) | (int(linear_prefix) << 8) | (MFN_CONV_BF16 if bf16 else 0)


def conv3x3_slices(buf_in: torch.Tensor, c_in0: int, Cin: int, packed: torch.Tensor, bias: Optional[torch.Tensor],
                   buf_out: torch.Tensor, c_out0: int, Cout: int, leaky_slope: float = 0.1, dilation: int = 1,
                   stride: int = 1, depth_to_space: bool = False, linear_prefix: int = 0, bf16: bool = False) -> None:
    """out = LeakyReLU(conv3x3(buf_in[:, c_in0:c_in0+Cin]) + bias) written to buf_out[:, c_out0:c_out0+Cout]; both buffers
    dense NCHW (they may be the same tensor: the dense block's concat buffer).  stride 2 (pad 1) = the pyramid's
    down-sampling convolutions: buf_out is then ((H-1)//2+1, (W-1)//2+1).  depth_to_space: the Cout = 4F conv channels
    are written as F channels of a (2H, 2W) image (sub-pixel phases; see conv_transpose4x4_pack).  linear_prefix: the first
    k output channels skip the activation (MFN_CONV_OUT_LINEAR_PREFIX).  bf16: one bf16 product per multiply-add
    (MFN_CONV_BF16: input and weights rounded once to bf16, fp32 accumulation) instead of the fp32-accurate split; the
    output stays fp32.  Inference only."""
    for t, nm in ((buf_in, "buf_in"), (buf_out, "buf_out")):
        if not (t.is_cuda and t.dtype == torch.float32 and t.is_contiguous() and t.dim() == 4):
            raise MaskflowError(f"conv3x3_slices: {nm} must be a contiguous CUDA float32 NCHW tensor")
    N, Cti, H, W = buf_in.shape
    OH, OW = (H - 1) // stride + 1, (W - 1) // stride + 1
    if depth_to_space:
        OH, OW = 2 * OH, 2 * OW
    Fo = Cout // 4 if depth_to_space else Cout        # channels written
    if buf_out.shape[0] != N or tuple(buf_out.shape[2:]) != (OH, OW):
        raise MaskflowError("conv3x3_slices: buffers disagree in N/H/W")
    Cto = buf_out.shape[1]
    if not (0 <= c_in0 and c_in0 + Cin <= Cti and 0 <= c_out0 and c_out0 + Fo <= Cto):
        raise MaskflowError("conv3x3_slices: channel slice out of range")
    if buf_in.data_ptr() == buf_out.data_ptr() and not (c_out0 + Cout <= c_in0 or c_in0 + Cin <= c_out0):
        raise MaskflowError("conv3x3_slices: input and output slices overlap")
    b = _chk(bias, "conv3x3_slices.bias", optional=True)
    _no_grad_path("conv3x3_slices", buf_in, b)
    xin = ctypes.c_void_p(buf_in.data_ptr() + 4 * c_in0 * H * W)
    xout = ctypes.c_void_p(buf_out.data_ptr() + 4 * c_out0 * OH * OW)
    # split-K scratch for the layers of the small pyramid levels (0 bytes = the library does not split this shape)
    ws_bytes = int(_lib.lib().mfn_conv3x3_workspace_bytes(N, Cin, H, W, Cout, int(stride), int(dilation)))
    ws = torch.empty(ws_bytes // 4, device=buf_in.device, dtype=torch.float32) if ws_bytes else None
    _call("mfn_conv3x3_forward_ws", buf_in.device, xin, Cti * H * W, _p(packed), _p(b), xout, Cto * OH * OW, N, Cin, H, W,
          Cout, int(stride), int(dilation), _out_mode(depth_to_space, linear_prefix, bf16), float(leaky_slope), _p(ws),
          ws_bytes)


class SplitAct:
    """An activation of `channels` channels in the split format the convolutions read with tensor copies
    (include/maskflow_b200.h, mfn_split_pack): per sample, the bf16 hi images of ceil(C/16)*2 groups of 8 channels, then
    their lo images, 16 bytes per (group, pixel); pad channels are zero.  bf16=True: a bf16 activation (mfn_bf16_pack),
    the hi images alone -- every value rounded once to bf16 -- read and written by the convolutions' bf16 mode.
    Writers: pack() and conv3x3_split()."""
    bf16 = False

    def __init__(self, N: int, channels: int, H: int, W: int, device, bf16: bool = False):
        self.channels = int(channels)
        self.bf16 = bool(bf16)
        self.buf = torch.empty((N, 1 if self.bf16 else 2, (self.channels + 15) // 16 * 2, H, W, 16), dtype=torch.uint8,
                               device=device)

    @property
    def shape(self):
        N, _, _, H, W, _ = self.buf.shape
        return N, self.channels, H, W

    def pack(self, src: torch.Tensor, c0: int) -> None:
        """Channels [c0, c0 + C) = the fp32 NCHW tensor src (C channels; c0 a multiple of 16)."""
        s = _chk(src, "SplitAct.pack.src")
        N, C, H, W = s.shape
        if (N, H, W) != (self.shape[0], self.shape[2], self.shape[3]):
            raise MaskflowError("SplitAct.pack: src disagrees in N/H/W")
        _call("mfn_bf16_pack" if self.bf16 else "mfn_split_pack", s.device, _p(s), C * H * W, N, C, H, W, _p(self.buf),
              self.channels, int(c0))

    def hi_lo(self):
        """(hi, lo) as fp32 (N, C, H, W) tensors: the two bf16 terms of every value (lo = zeros for a bf16 activation)."""
        N, C, H, W = self.shape
        P = self.buf.shape[1]
        t = self.buf.view(torch.bfloat16).view(N, P, -1, H, W, 8).permute(0, 1, 2, 5, 3, 4).reshape(N, P, -1, H, W)
        hi = t[:, 0, :C].float()
        return hi, (t[:, 1, :C].float() if P == 2 else torch.zeros_like(hi))


def conv3x3_split(x: SplitAct, c_in0: int, Cin: int, packed: torch.Tensor, bias: Optional[torch.Tensor], Cout: int,
                  leaky_slope: float = 0.1, dilation: int = 1, out: Optional[torch.Tensor] = None,
                  out_split: Optional[SplitAct] = None, out_c0: int = 0, depth_to_space: bool = False,
                  linear_prefix: int = 0, bf16: bool = False) -> None:
    """conv3x3_slices reading channels [c_in0, c_in0 + Cin) of a split activation (c_in0 a multiple of 16).  Output: the
    fp32 NCHW (or depth-to-space) tensor `out`, or -- out_split given -- channels out_c0.. of that split activation, the
    linear_prefix channels (even) going to the fp32 (N, linear_prefix, H, W) `out`.  Bit-identical to conv3x3_slices on
    the same values.  bf16: the bf16 mode (see conv3x3_slices); x and out_split must then be bf16 activations
    (SplitAct(..., bf16=True)), and must not be otherwise.  Inference only."""
    for a, nm in ((x, "x"), (out_split, "out_split")):
        if a is not None and a.bf16 != bool(bf16):
            raise MaskflowError(f"conv3x3_split: {nm} is a {'bf16' if a.bf16 else 'split'} activation but bf16={bool(bf16)}")
    N, Cx, H, W = x.shape
    if not (0 <= c_in0 and c_in0 + Cin <= Cx):
        raise MaskflowError("conv3x3_split: channel slice out of range")
    if out is not None:
        f = Cout // 4 if depth_to_space else (linear_prefix if out_split is not None else Cout)
        s = 2 if depth_to_space else 1
        if not (out.is_cuda and out.dtype == torch.float32 and out.is_contiguous() and out.shape == (N, f, s * H, s * W)):
            raise MaskflowError(f"conv3x3_split: out must be a contiguous CUDA float32 tensor of shape {(N, f, s * H, s * W)}")
    if out_split is not None and (out_split.shape[0], out_split.shape[2], out_split.shape[3]) != (N, H, W):
        raise MaskflowError("conv3x3_split: out_split disagrees in N/H/W")
    if out_split is not None and out_split.buf.data_ptr() == x.buf.data_ptr():
        # the input is read in whole 16-channel groups, the output written in them
        r0, r1 = c_in0, -(-(c_in0 + Cin) // 16) * 16
        w0, w1 = out_c0, out_c0 + Cout - linear_prefix
        if not (w1 <= r0 or r1 <= w0):
            raise MaskflowError("conv3x3_split: input and output slices overlap")
    b = _chk(bias, "conv3x3_split.bias", optional=True)
    _no_grad_path("conv3x3_split", x.buf, b)
    ws_bytes = int(_lib.lib().mfn_conv3x3_workspace_bytes(N, Cin, H, W, Cout, 1, int(dilation)))
    ws = torch.empty(ws_bytes // 4, device=x.buf.device, dtype=torch.float32) if ws_bytes else None
    _call("mfn_conv3x3_forward_split", x.buf.device, _p(x.buf), Cx, int(c_in0), _p(packed), _p(b), _p(out), 0,
          _p(out_split.buf if out_split is not None else None), out_split.channels if out_split is not None else 0,
          int(out_c0), N, Cin, H, W, Cout, int(dilation), _out_mode(depth_to_space, linear_prefix, bf16),
          float(leaky_slope), _p(ws), ws_bytes)


def conv_transpose4x4_as_conv3x3(weight: torch.Tensor) -> torch.Tensor:
    """nn.ConvTranspose2d(Cin, F, kernel 4, stride 2, pad 1) (the decoder's `upfeat` layers, network/MaskFlownet.py:225 ...)
    re-arranged as the weight (4F, Cin, 3, 3) of a 3x3 convolution followed by depth-to-space: output pixel (2y+py, 2x+px)
    only touches inputs (y+dy, x+dx) with dy in {0, -1} (py = 0) or {0, +1} (py = 1), through kernel row ky = py + 1 - 2 dy
    (likewise columns).  Conv channel (2 py + px) * F + f; the five unused taps of every phase are zero.  Pure tensor
    algebra (any device) -- checked on the CPU in tests/test_host_logic.py."""
    w = weight.detach()
    Cin, F, kh, kw = w.shape
    if (kh, kw) != (4, 4):
        raise MaskflowError("conv_transpose4x4_as_conv3x3: weight must be (Cin, F, 4, 4)")
    w3 = torch.zeros((4 * F, Cin, 3, 3), device=w.device, dtype=torch.float32)
    for py in range(2):
        for px in range(2):
            ph = 2 * py + px
            for dy in ((0, -1) if py == 0 else (0, 1)):
                for dx in ((0, -1) if px == 0 else (0, 1)):
                    ky, kx = py + 1 - 2 * dy, px + 1 - 2 * dx
                    w3[ph * F:(ph + 1) * F, :, dy + 1, dx + 1] = w[:, :, ky, kx].t()
    return w3


def conv_transpose4x4_pack(weight: torch.Tensor) -> torch.Tensor:
    """Packed weight image of conv_transpose4x4_as_conv3x3(weight) for conv3x3_slices(..., depth_to_space=True)."""
    return conv3x3_pack(conv_transpose4x4_as_conv3x3(_chk(weight, "conv_transpose4x4_pack.weight")))


def conv3x3(x: torch.Tensor, packed: torch.Tensor, bias: Optional[torch.Tensor], Cout: int, leaky_slope: float = 0.1,
            dilation: int = 1, stride: int = 1, bf16: bool = False):
    """3x3 convolution, padding = dilation, stride 1 (decoder / context network) or 2 (pyramid), + LeakyReLU.  bf16: the
    bf16 mode of conv3x3_slices."""
    x = _chk(x, "conv3x3.x")
    out = torch.empty((x.shape[0], Cout, (x.shape[2] - 1) // stride + 1, (x.shape[3] - 1) // stride + 1), device=x.device,
                      dtype=torch.float32)
    conv3x3_slices(x, 0, x.shape[1], packed, bias, out, 0, Cout, leaky_slope, dilation, stride, bf16=bf16)
    return out


class _Conv3x3TrainFn(torch.autograd.Function):
    """Training-mode 3x3 convolution (+ bias + LeakyReLU): FORWARD on the wgmma kernel (the same launch inference uses),
    BACKWARD through aten.convolution_backward (cuDNN dgrad / wgrad -- this library has no convolution backward kernels,
    cuDNN's backward).  The activation's backward uses the saved OUTPUT (y > 0  <=>  pre-activation > 0 for slope > 0)."""

    @staticmethod
    def forward(ctx, x, weight, bias, packed, slope, dilation, stride):
        y = conv3x3(x, packed, bias, weight.shape[0], slope, dilation, stride)      # grad mode is off inside forward()
        ctx.save_for_backward(x, weight, y)
        ctx.cfg = (float(slope), int(dilation), int(stride), bias is not None)
        return y

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, g):
        x, weight, y = ctx.saved_tensors
        slope, dilation, stride, has_bias = ctx.cfg
        if slope != 1.0:
            g = torch.where(y > 0, g, g * slope)
        gx, gw, gb = torch.ops.aten.convolution_backward(
            g.contiguous(), x, weight, [weight.shape[0]] if has_bias else None, [stride, stride], [dilation, dilation],
            [dilation, dilation], False, [0, 0], 1,
            [ctx.needs_input_grad[0], ctx.needs_input_grad[1], has_bias and ctx.needs_input_grad[2]])
        return gx, gw, (gb if has_bias else None), None, None, None, None


def conv3x3_train(x: torch.Tensor, weight: torch.Tensor, bias: Optional[torch.Tensor], packed: torch.Tensor,
                  leaky_slope: float = 0.1, dilation: int = 1, stride: int = 1) -> torch.Tensor:
    """LeakyReLU(conv3x3(x, weight) + bias) with autograd: tensor-core forward, cuDNN backward (see _Conv3x3TrainFn).
    `packed` = conv3x3_pack(weight) for the CURRENT value of weight (network._packed re-packs when the parameter's version
    changes, i.e. after every optimizer step)."""
    x = _chk(x, "conv3x3_train.x")
    if weight.dim() != 4 or tuple(weight.shape[2:]) != (3, 3) or weight.shape[1] != x.shape[1]:
        raise MaskflowError(f"conv3x3_train: weight {tuple(weight.shape)} does not fit x {tuple(x.shape)}")
    return _Conv3x3TrainFn.apply(x, weight, bias, packed, leaky_slope, dilation, stride)


# ----------------------------------------------------------------------------------------------------------
# Pre / post-processing around the network (row N3)
# ----------------------------------------------------------------------------------------------------------
def padded_size(H: int, W: int, resize=None):
    """Network input size for an (H, W) image: the next multiples of 64 (network/pipeline.py:122-124), or `resize`."""
    if resize is not None:
        return int(resize[0]), int(resize[1])
    return H + (64 - H % 64) % 64, W + (64 - W % 64) % 64


def preprocess(img1: torch.Tensor, img2: torch.Tensor, out_hw=None):
    """/255 (uint8 input) -> centralize -> BilinearResize2D to out_hw: what PipelineFlownet.predict + do_batch_mx do before
    the network (network/pipeline.py:206-212, 85-87, 117-130).  Returns (im1, im2, rgb_mean (N,C,1,1)).  Forward only.
    im1 and im2 are the two halves of one (2N, C, OH, OW) buffer, which the network's shared pyramid reads as one batch
    without a copy."""
    for t, nm in ((img1, "img1"), (img2, "img2")):
        if not (t.is_cuda and t.is_contiguous() and t.dim() == 4 and t.dtype in (torch.uint8, torch.float32)):
            raise MaskflowError(f"preprocess: {nm} must be a contiguous CUDA uint8 / float32 NCHW tensor")
    if img1.shape != img2.shape or img1.dtype != img2.dtype:
        raise MaskflowError("preprocess: img1 and img2 must agree in shape and dtype")
    _no_grad_path("preprocess", img1, img2)
    N, C, H, W = img1.shape
    OH, OW = (H, W) if out_hw is None else (int(out_hw[0]), int(out_hw[1]))
    pair = torch.empty((2 * N, C, OH, OW), device=img1.device, dtype=torch.float32)
    o1, o2 = pair[:N], pair[N:]
    mean = torch.empty((N, C, 1, 1), device=img1.device, dtype=torch.float32)
    args = (_p(img1), _p(img2), 1 if img1.dtype == torch.uint8 else 0, _p(o1), _p(o2), _p(mean), N, C, H, W, OH, OW)
    if deterministic():
        nb = det_workspace_bytes("preprocess", N, C, H, W)
        _call("mfn_preprocess_forward_det", img1.device, *args, _p(_det_ws(nb, img1.device)), nb)
    else:
        _call("mfn_preprocess_forward", img1.device, *args)
    return o1, o2, mean


def postprocess(pred: torch.Tensor, H: int, W: int, flip_channels: bool = True, is_flow: bool = True) -> torch.Tensor:
    """Upsample(4) -> BilinearResize2D back to (H, W) (flow rescaled per channel) -> NHWC -> (y,x) to (x,y) flip: what
    do_batch + predict do after the network (network/pipeline.py:137-141, 217-218).  pred (N,ch,Hq,Wq) -> (N,H,W,ch)."""
    p = _chk(pred, "postprocess.pred")
    _no_grad_path("postprocess", p)
    N, CH, Hq, Wq = p.shape
    out = torch.empty((N, H, W, CH), device=p.device, dtype=torch.float32)
    _call("mfn_postprocess_forward", p.device, _p(p), _p(out), N, CH, Hq, Wq, int(H), int(W), 1 if flip_channels else 0,
          1 if is_flow else 0)
    return out


def flow_to_color(flow_xy: torch.Tensor, max_radius: Optional[float] = None, bgr: bool = False):
    """Middlebury colour coding (flow_vis.flow_to_color, what predict_new_data.py writes) of an (x,y) flow in pixels, the
    layout postprocess returns: (N,H,W,2) -> (rgb uint8 (N,H,W,3), rad_max (N,)); an (H,W,2) flow gives (H,W,3) and a
    0-d rad_max.  max_radius None: each sample is normalised by its own largest radius (the reference); a positive
    value fixes the scale, so that colours stay comparable across the frames of a video.  rad_max is the radius used.
    Channels R,G,B, or B,G,R with bgr (for cv2).  Forward only."""
    f = _chk(flow_xy, "flow_to_color.flow_xy")
    if f.dim() not in (3, 4) or f.shape[-1] != 2:
        raise MaskflowError(f"flow_to_color: expected an (N,H,W,2) or (H,W,2) flow, got {tuple(f.shape)}")
    if max_radius is not None and not (0.0 < float(max_radius) < float("inf")):
        raise MaskflowError(f"flow_to_color: max_radius must be positive and finite, got {max_radius}")
    _no_grad_path("flow_to_color", f)
    f4 = f if f.dim() == 4 else f.unsqueeze(0)
    N, H, W, _ = f4.shape
    rgb = torch.empty((N, H, W, 3), device=f.device, dtype=torch.uint8)
    rad_max = torch.empty((N,), device=f.device, dtype=torch.float32)
    _call("mfn_flow_to_color", f.device, _p(f4), _p(rgb), _p(rad_max), N, H, W,
          float(max_radius) if max_radius is not None else 0.0, 1 if bgr else 0)
    return (rgb, rad_max) if f.dim() == 4 else (rgb[0], rad_max[0])


def flow_consistency(flow_fw: torch.Tensor, flow_bw: torch.Tensor, alpha: float = 0.01, beta: float = 0.5):
    """Forward-backward consistency check (Sundaram, Brox and Keutzer, ECCV 2010) of the flows image 1 -> image 2
    (flow_fw) and image 2 -> image 1 (flow_bw), (x,y) in pixels, the layout postprocess returns: (N,H,W,2) ->
    (occ_fw, occ_bw) uint8 (N,H,W), 1 where a pixel of image 1 (occ_fw) / image 2 (occ_bw) has no consistent match in the
    other image: its target leaves the frame, or |w + w_other(target)|^2 > alpha (|w|^2 + |w_other(target)|^2) + beta
    (NaN or inf anywhere: 1).  An (H,W,2) pair gives (H,W) masks.  Defaults: the paper's constants.  Forward only (include/maskflow_b200.h)."""
    for t, nm in ((flow_fw, "flow_fw"), (flow_bw, "flow_bw")):
        if not isinstance(t, torch.Tensor) or not t.is_cuda:
            raise MaskflowError(f"flow_consistency: {nm} must be a CUDA tensor; the hot path has no CPU implementation")
        if t.dtype != torch.float32 or not t.is_contiguous():
            raise MaskflowError(f"flow_consistency: {nm} must be a contiguous float32 tensor")
        if t.dim() not in (3, 4) or t.shape[-1] != 2:
            raise MaskflowError(f"flow_consistency: expected an (N,H,W,2) or (H,W,2) {nm}, got {tuple(t.shape)}")
    if flow_fw.shape != flow_bw.shape or flow_fw.device != flow_bw.device:
        raise MaskflowError(f"flow_consistency: flow_fw {tuple(flow_fw.shape)} and flow_bw {tuple(flow_bw.shape)} differ")
    inf = float("inf")
    if not (0.0 <= float(alpha) < inf and 0.0 <= float(beta) < inf):
        raise MaskflowError(f"flow_consistency: alpha and beta must be finite and non-negative, got {alpha}, {beta}")
    _no_grad_path("flow_consistency", flow_fw, flow_bw)
    fw = flow_fw if flow_fw.dim() == 4 else flow_fw.unsqueeze(0)
    bw = flow_bw if flow_bw.dim() == 4 else flow_bw.unsqueeze(0)
    N, H, W, _ = fw.shape
    occ_fw = torch.empty((N, H, W), device=fw.device, dtype=torch.uint8)
    occ_bw = torch.empty((N, H, W), device=fw.device, dtype=torch.uint8)
    _call("mfn_flow_consistency", fw.device, _p(fw), _p(bw), _p(occ_fw), _p(occ_bw), N, H, W, float(alpha), float(beta))
    return (occ_fw, occ_bw) if flow_fw.dim() == 4 else (occ_fw[0], occ_bw[0])


def _interp_times(times, who: str):
    """times -> a tuple of floats, each in (0,1)."""
    try:
        ts = tuple(float(t) for t in times)
    except TypeError:               # a single time
        ts = (float(times),)
    if not ts:
        raise MaskflowError(f"{who}: at least one time is required")
    for t in ts:
        if not 0.0 < t < 1.0:
            raise MaskflowError(f"{who}: every time must lie in (0,1), got {t}")
    return ts


def interpolate_frames(img0: torch.Tensor, img1: torch.Tensor, flow_fw: torch.Tensor, flow_bw: torch.Tensor,
                       occ_fw: torch.Tensor, occ_bw: torch.Tensor, times, occ_weight: float = 0.01) -> torch.Tensor:
    """In-between frames of image pairs by occlusion-weighted forward splatting of both images along their flows
    (include/maskflow_b200.h, mfn_interpolate_frames).  img0, img1 (N,H,W,3) uint8, any channel order (the layout of the
    video predictor's frame buffer); flow_fw (img0 -> img1) and flow_bw (img1 -> img0) (N,H,W,2) float32 (x,y) pixels, the
    layout postprocess and network.predict_bidirectional return; occ_fw, occ_bw (N,H,W) uint8 from flow_consistency.
    times: one time or a sequence, each in (0,1) (0 = img0).  At time t each pixel of img0 moves by t * flow_fw with weight
    (1 - t), each of img1 by (1 - t) * flow_bw with weight t, occluded ones weighted by occ_weight (in [0,1]); pixels no
    source reaches take the blend (1 - t) img0 + t img1.  Returns (N,T,H,W,3) uint8; (H,W,...) inputs give (T,H,W,3).
    Bit-reproducible.  Forward only."""
    ts = _interp_times(times, "interpolate_frames")
    if not (0.0 <= float(occ_weight) <= 1.0):
        raise MaskflowError(f"interpolate_frames: occ_weight must lie in [0,1], got {occ_weight}")
    args = ((img0, "img0", torch.uint8, 3), (img1, "img1", torch.uint8, 3), (flow_fw, "flow_fw", torch.float32, 2),
            (flow_bw, "flow_bw", torch.float32, 2), (occ_fw, "occ_fw", torch.uint8, None), (occ_bw, "occ_bw", torch.uint8, None))
    batched = isinstance(img0, torch.Tensor) and img0.dim() == 4
    lead = None
    for t, nm, dtype, last in args:
        if not isinstance(t, torch.Tensor) or not t.is_cuda:
            raise MaskflowError(f"interpolate_frames: {nm} must be a CUDA tensor; the hot path has no CPU implementation")
        if t.dtype != dtype or not t.is_contiguous():
            raise MaskflowError(f"interpolate_frames: {nm} must be a contiguous {dtype} tensor")
        dims = (4 if batched else 3) - (last is None)
        if t.dim() != dims or (last is not None and t.shape[-1] != last):
            want = ("(N,H,W" if batched else "(H,W") + (f",{last})" if last is not None else ")")
            raise MaskflowError(f"interpolate_frames: expected {nm} of shape {want}, got {tuple(t.shape)}")
        ld = tuple(t.shape[:dims if last is None else dims - 1])
        if lead is None:
            lead, dev = ld, t.device
        elif ld != lead or t.device != dev:
            raise MaskflowError(f"interpolate_frames: {nm} {tuple(t.shape)} on {t.device} does not match img0 "
                                f"{tuple(img0.shape)} on {img0.device}")
    _no_grad_path("interpolate_frames", flow_fw, flow_bw)
    if not batched:
        img0, img1, flow_fw, flow_bw, occ_fw, occ_bw = (t.unsqueeze(0) for t in (img0, img1, flow_fw, flow_bw, occ_fw, occ_bw))
    N, H, W, _ = img0.shape
    out = torch.empty((N, len(ts), H, W, 3), device=dev, dtype=torch.uint8)
    nb = int(_lib.lib().mfn_interpolate_frames_workspace_bytes(N, H, W))
    ws = torch.empty(nb, dtype=torch.uint8, device=dev)
    times_host = (ctypes.c_float * len(ts))(*ts)
    _call("mfn_interpolate_frames", dev, _p(img0), _p(img1), _p(flow_fw), _p(flow_bw), _p(occ_fw), _p(occ_bw), _p(out),
          _p(ws), nb, N, H, W, ctypes.cast(times_host, ctypes.c_void_p), len(ts), float(occ_weight))
    return out if batched else out[0]


# ----------------------------------------------------------------------------------------------------------
# Video stabilisation (csrc/stabilize.cu)
# ----------------------------------------------------------------------------------------------------------
# Defaults of the robust fit, from the robustness scene of tests/test_stabilize.py (a known camera map, 0.3 px noise, a
# square over 30 % of the frame moving 14 px relative to it): the largest error at the frame corners was 0.126 px with
# 8 iterations at sigma 1, 0.064 px with 8 at 0.5, 0.054 px with 10 at 0.5 and 0.043 px with 10 at 0.25; with the square
# moving 5.8 px: 0.51, 0.19, 0.14 and 0.099 px.  Cauchy weights never drop an outlier completely, so a smaller sigma and
# more iterations help; sigma 0.5 keeps inliers with the flow noise of trained networks (about 0.3-0.5 px) weighted.
AFFINE_ITERATIONS, AFFINE_SIGMA = 10, 0.5


def _stab_tensor(t, nm: str, dtype, last, who: str) -> torch.Tensor:
    if not isinstance(t, torch.Tensor) or not t.is_cuda:
        raise MaskflowError(f"{who}: {nm} must be a CUDA tensor; the hot path has no CPU implementation")
    if t.dtype != dtype or not t.is_contiguous():
        raise MaskflowError(f"{who}: {nm} must be a contiguous {dtype} tensor")
    if t.dim() != 4 or t.shape[-1] != last:
        raise MaskflowError(f"{who}: expected {nm} of shape (N,H,W,{last}), got {tuple(t.shape)}")
    return t


def check_affine_args(iterations, sigma, who: str) -> None:
    if not (isinstance(iterations, int) and not isinstance(iterations, bool) and iterations >= 1):
        raise MaskflowError(f"{who}: iterations must be an integer >= 1, got {iterations!r}")
    try:
        good = 0.0 < float(sigma) < float("inf")
    except (TypeError, ValueError):
        good = False
    if not good:
        raise MaskflowError(f"{who}: sigma must be positive and finite, got {sigma!r}")


def affine_motion(flow: torch.Tensor, iterations: int = AFFINE_ITERATIONS, sigma: float = AFFINE_SIGMA,
                  want_residual: bool = False):
    """The camera's motion between the two images of each pair: a robust affine fit to the flow (include/maskflow_b200.h,
    mfn_affine_motion).  flow (N,H,W,2) float32 (x,y) pixels, the layout postprocess and network.predict return.  Pixels
    whose target leaves the frame (or is not finite) are left out; iteration 0 is plain least squares, each later one
    reweights every pixel by the Cauchy weight 1 / (1 + (r / sigma_k)^2) of its residual r under the previous fit, with
    sigma_k = sigma 2^max(0, 4-k) annealed from 8 sigma down to sigma (pixels).
    Returns (affine (N,2,3) float64 with affine @ [x,y,1] ~ [x,y] + flow[y,x], ok (N,) bool[, residual (N,H,W) float32]):
    ok is False where the last solve was ill conditioned (too few valid pixels, or all of them on one line), and affine is
    then the identity.  residual: |affine p - q| in pixels under the final fit, NaN where the pixel was left out.
    Bit-reproducible; a sample's result does not depend on the batch it is in.  Forward only."""
    check_affine_args(iterations, sigma, "affine_motion")
    f = _stab_tensor(flow, "flow", torch.float32, 2, "affine_motion")
    _no_grad_path("affine_motion", f)
    N, H, W, _ = f.shape
    dev = f.device
    affine = torch.empty((N, 2, 3), device=dev, dtype=torch.float64)
    ok = torch.empty((N,), device=dev, dtype=torch.uint8)
    residual = torch.empty((N, H, W), device=dev, dtype=torch.float32) if want_residual else None
    nb = int(_lib.lib().mfn_affine_motion_workspace_bytes(N, H, W))
    ws = torch.empty(nb, dtype=torch.uint8, device=dev)
    _call("mfn_affine_motion", dev, _p(f), _p(affine), _p(ok), _p(residual), _p(ws), nb, N, H, W, int(iterations),
          float(sigma))
    return (affine, ok.bool(), residual) if want_residual else (affine, ok.bool())


def warp_frames_affine(frames: torch.Tensor, M: torch.Tensor) -> torch.Tensor:
    """Each frame warped by its affine map (include/maskflow_b200.h, mfn_warp_frames_affine): out[n](o) = frames[n]
    sampled bilinearly at M[n] @ [o, 1], the position clamped to the frame (the border is replicated), rounded to nearest.
    frames (N,H,W,3) uint8, any channel order; M (N,2,3) float64 on the same device, output pixel -> source position.
    Returns (N,H,W,3) uint8.  Deterministic."""
    fr = _stab_tensor(frames, "frames", torch.uint8, 3, "warp_frames_affine")
    if not isinstance(M, torch.Tensor) or M.device != fr.device:
        raise MaskflowError(f"warp_frames_affine: M must be a tensor on {fr.device}")
    if M.dtype != torch.float64 or not M.is_contiguous() or tuple(M.shape) != (fr.shape[0], 2, 3):
        raise MaskflowError(f"warp_frames_affine: M must be a contiguous float64 tensor of shape ({fr.shape[0]},2,3), "
                            f"got {M.dtype} {tuple(M.shape)}")
    N, H, W, _ = fr.shape
    out = torch.empty_like(fr)
    _call("mfn_warp_frames_affine", fr.device, _p(fr), _p(M), _p(out), N, H, W)
    return out


# ----------------------------------------------------------------------------------------------------------
# Moving-object segmentation (csrc/motionseg.cu)
# ----------------------------------------------------------------------------------------------------------
# Defaults, from the synthetic scene of tests/test_motion_segment.py (README, "Moving-object segmentation").
SEG_TAU_LO, SEG_TAU_HI, SEG_MIN_AREA, SEG_MAX_OBJECTS = 1.0, 2.0, 64, 255


def check_segment_args(tau_lo, tau_hi, min_area, max_objects, who: str) -> None:
    try:
        lo, hi = float(tau_lo), float(tau_hi)
    except (TypeError, ValueError):
        raise MaskflowError(f"{who}: tau_lo and tau_hi must be numbers, got {tau_lo!r}, {tau_hi!r}") from None
    inf = float("inf")
    lo, hi = (torch.tensor(v, dtype=torch.float32).item() for v in (lo, hi))     # the kernel compares in float32
    if not (-inf < lo <= hi < inf):
        raise MaskflowError(f"{who}: tau_lo and tau_hi must be finite with tau_lo <= tau_hi, got {tau_lo}, {tau_hi}")
    if not (isinstance(min_area, int) and not isinstance(min_area, bool) and min_area >= 1):
        raise MaskflowError(f"{who}: min_area must be an integer >= 1, got {min_area!r}")
    if not (isinstance(max_objects, int) and not isinstance(max_objects, bool) and 1 <= max_objects <= 255):
        raise MaskflowError(f"{who}: max_objects must be an integer in [1,255], got {max_objects!r}")


def segment_motion(res_a=None, occ_a=None, res_b=None, occ_b=None, flow_a=None, affine_a=None, tau_lo: float = SEG_TAU_LO,
                   tau_hi: float = SEG_TAU_HI, min_area: int = SEG_MIN_AREA, max_objects: int = SEG_MAX_OBJECTS,
                   shape=None):
    """The objects that move relative to the camera in each of N frames (include/maskflow_b200.h,
    mfn_motion_segment).  Frame n takes up to two sides: side a, the forward direction of the pair (n, n+1) --
    res_a (N,H,W) float32, affine_motion's residual of the forward flow; occ_a (N,H,W) uint8, its flow_consistency mask;
    flow_a (N,H,W,2) float32, the forward flow; affine_a (N,2,3) float64, its fit -- and side b, the backward direction of
    the pair (n-1, n): res_b, occ_b.  A side is given whole or not at all; with neither, `shape` = (N,H,W) gives empty
    frames.  Per pixel s = the smaller of the defined residuals (finite and not occluded); the 8-connected components of
    s >= tau_lo that reach s >= tau_hi somewhere and cover at least min_area pixels are the objects, numbered 1, 2, ...
    in raster order of their first pixel, up to max_objects (at most 255).
    Returns (labels (N,H,W) uint8, 0 = background; objects (N,max_objects,10) float64, rows (area, x0, y0, x1, y1, cx,
    cy, peak, dx, dy) for the first count[n] labels, 0 past them -- dx, dy the mean camera-relative displacement
    p + flow_a(p) - A p where side a is defined, NaN where it is nowhere; count (N,) int32; dropped (N,) int32, the objects
    past max_objects).  Bit-reproducible and capture-safe.  Forward only."""
    who = "segment_motion"
    check_segment_args(tau_lo, tau_hi, min_area, max_objects, who)
    side_a, side_b = (res_a, occ_a, flow_a, affine_a), (res_b, occ_b)
    have_a, have_b = any(t is not None for t in side_a), any(t is not None for t in side_b)
    if have_a and any(t is None for t in side_a):
        raise MaskflowError(f"{who}: res_a, occ_a, flow_a and affine_a go together")
    if have_b and any(t is None for t in side_b):
        raise MaskflowError(f"{who}: res_b and occ_b go together")
    args = []
    if have_a:
        args += [(res_a, "res_a", torch.float32, None), (occ_a, "occ_a", torch.uint8, None),
                 (flow_a, "flow_a", torch.float32, 2)]
    if have_b:
        args += [(res_b, "res_b", torch.float32, None), (occ_b, "occ_b", torch.uint8, None)]
    lead = dev = None
    for t, nm, dtype, last in args:
        if not isinstance(t, torch.Tensor) or not t.is_cuda:
            raise MaskflowError(f"{who}: {nm} must be a CUDA tensor; the hot path has no CPU implementation")
        if t.dtype != dtype or not t.is_contiguous():
            raise MaskflowError(f"{who}: {nm} must be a contiguous {dtype} tensor")
        if t.dim() != (3 if last is None else 4) or (last is not None and t.shape[-1] != last):
            raise MaskflowError(f"{who}: expected {nm} of shape (N,H,W{'' if last is None else ',2'}), got {tuple(t.shape)}")
        ld = tuple(t.shape[:3])
        if lead is None:
            lead, dev = ld, t.device
        elif ld != lead or t.device != dev:
            raise MaskflowError(f"{who}: {nm} {tuple(t.shape)} on {t.device} does not match {lead} on {dev}")
    if have_a:
        if not isinstance(affine_a, torch.Tensor) or affine_a.device != dev or affine_a.dtype != torch.float64 or \
                not affine_a.is_contiguous() or tuple(affine_a.shape) != (lead[0], 2, 3):
            raise MaskflowError(f"{who}: affine_a must be a contiguous float64 tensor of shape ({lead[0]},2,3) on {dev}")
        _no_grad_path(who, res_a, flow_a)
    if have_b:
        _no_grad_path(who, res_b)
    if lead is None:
        if shape is None or len(shape) != 3 or min(int(v) for v in shape) < 1:
            raise MaskflowError(f"{who}: without either side, shape must be (N,H,W), got {shape!r}")
        lead, dev = tuple(int(v) for v in shape), torch.device("cuda", torch.cuda.current_device())
    N, H, W = lead
    labels = torch.empty((N, H, W), device=dev, dtype=torch.uint8)
    objects = torch.empty((N, max_objects, 10), device=dev, dtype=torch.float64)
    count = torch.empty((N,), device=dev, dtype=torch.int32)
    dropped = torch.empty((N,), device=dev, dtype=torch.int32)
    nb = int(_lib.lib().mfn_motion_segment_workspace_bytes(N, H, W))
    ws = torch.empty(nb, dtype=torch.uint8, device=dev)
    _call("mfn_motion_segment", dev, _p(res_a), _p(occ_a), _p(res_b), _p(occ_b), _p(flow_a), _p(affine_a), _p(labels),
          _p(objects), _p(count), _p(dropped), _p(ws), nb, N, H, W, float(tau_lo), float(tau_hi), int(min_area),
          int(max_objects))
    return labels, objects, count, dropped


# ----------------------------------------------------------------------------------------------------------
# Video denoising (csrc/denoise.cu)
# ----------------------------------------------------------------------------------------------------------
# Defaults, from the sweep over the synthetic scene of tests/test_denoise.py through the oracle (README, "Video
# denoising"): R neighbours on each side, a (2 DENOISE_PATCH + 1)^2 patch, h = DENOISE_H sigma.
DENOISE_RADIUS, DENOISE_PATCH, DENOISE_H = 2, 1, 0.7
DENOISE_MAX_PATCH = 8       # the kernel's shared-memory bound on the patch radius
NOISE_FLOOR = 0.5           # estimate_noise never returns less (grey levels)


def _positive_finite(v) -> bool:
    try:
        return 0.0 < float(v) < float("inf")
    except (TypeError, ValueError):
        return False


def _int_at_least(v, lo) -> bool:
    return isinstance(v, int) and not isinstance(v, bool) and v >= lo


def check_denoise_args(radius, sigma, h, patch, alpha, beta, who: str, sigma_optional: bool = False) -> None:
    if not _int_at_least(radius, 0):
        raise MaskflowError(f"{who}: radius must be an integer >= 0, got {radius!r}")
    if not (_int_at_least(patch, 0) and patch <= DENOISE_MAX_PATCH):
        raise MaskflowError(f"{who}: patch must be an integer in [0,{DENOISE_MAX_PATCH}], got {patch!r}")
    if not (sigma is None and sigma_optional) and not _positive_finite(sigma):
        raise MaskflowError(f"{who}: sigma must be positive and finite, got {sigma!r}")
    if not _positive_finite(h):
        raise MaskflowError(f"{who}: h must be positive and finite, got {h!r}")
    if not (_finite_nonneg(alpha) and _finite_nonneg(beta)):
        raise MaskflowError(f"{who}: alpha and beta must be finite and non-negative, got {alpha!r}, {beta!r}")


def denoise_frames(frames: torch.Tensor, flow_fw: torch.Tensor, flow_bw: torch.Tensor, radius: int, sigma: float,
                   h: float = DENOISE_H, patch: int = DENOISE_PATCH, alpha: float = 0.01, beta: float = 0.5,
                   t0: int = 0, n: Optional[int] = None, t_lo: int = 0, t_hi: Optional[int] = None,
                   out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Frames t0 .. t0+n-1 of a video, each averaged with up to `radius` neighbours on each side aligned along the
    chained flow and weighted by a patch distance (include/maskflow_b200.h, mfn_denoise_frames).
    frames (S,H,W,3) uint8, any channel order, a ring: frame t in slot t % S.  flow_fw, flow_bw (S,H,W,2) float32 (x,y)
    pixels, rings: slot t % S holds pair (t, t+1), flow_fw t -> t+1 and flow_bw t+1 -> t (the layout
    network.predict_bidirectional returns).  The video's frames are [t_lo, t_hi] (default t_lo + S - 1): a plain clip of
    T frames is S = T with the defaults.  A chain stops where its target leaves the frame or the forward-backward check
    (alpha, beta) fails.  Neighbour k of pixel p gets the weight exp(-max(d2 - 2 sigma^2, 0) / (h sigma)^2), d2 the mean
    squared colour difference over the (2 patch + 1)^2 patch around p where the neighbour is defined; sigma is the noise
    level in grey levels (estimate_noise).  n defaults to t_hi - t0 + 1.  Returns (n,H,W,3) uint8 (into `out` when
    given).  Deterministic and capture-safe.  Forward only."""
    who = "denoise_frames"
    check_denoise_args(radius, sigma, h, patch, alpha, beta, who)
    fr = _stab_tensor(frames, "frames", torch.uint8, 3, who)
    fw = _stab_tensor(flow_fw, "flow_fw", torch.float32, 2, who)
    bw = _stab_tensor(flow_bw, "flow_bw", torch.float32, 2, who)
    S, H, W, _ = fr.shape
    for t, nm in ((fw, "flow_fw"), (bw, "flow_bw")):
        if tuple(t.shape[:3]) != (S, H, W) or t.device != fr.device:
            raise MaskflowError(f"{who}: {nm} {tuple(t.shape)} on {t.device} does not match frames {tuple(fr.shape)} "
                                f"on {fr.device}")
    _no_grad_path(who, fw, bw)
    for v, nm in ((t0, "t0"), (t_lo, "t_lo")):
        if not _int_at_least(v, 0):
            raise MaskflowError(f"{who}: {nm} must be an integer >= 0, got {v!r}")
    t_hi = t_lo + S - 1 if t_hi is None else t_hi
    n = t_hi - t0 + 1 if n is None else n
    if not (_int_at_least(t_hi, 0) and _int_at_least(n, 1)):
        raise MaskflowError(f"{who}: t_hi must be an integer >= 0 and n >= 1, got {t_hi!r}, {n!r}")
    if not t_lo <= t0 <= t0 + n - 1 <= t_hi:
        raise MaskflowError(f"{who}: frames {t0}..{t0 + n - 1} lie outside the video's frames {t_lo}..{t_hi}")
    span = min(t_hi, t0 + n - 1 + radius) - max(t_lo, t0 - radius) + 1
    if span > S:
        raise MaskflowError(f"{who}: the windows span {span} frames, more than the ring's {S} slots")
    if out is None:
        out = torch.empty((n, H, W, 3), dtype=torch.uint8, device=fr.device)
    elif not (isinstance(out, torch.Tensor) and out.dtype == torch.uint8 and out.is_contiguous() and
              tuple(out.shape) == (n, H, W, 3) and out.device == fr.device):
        raise MaskflowError(f"{who}: out must be a contiguous uint8 tensor of shape ({n},{H},{W},3) on {fr.device}")
    _call("mfn_denoise_frames", fr.device, _p(fr), _p(fw), _p(bw), _p(out), S, H, W, int(t0), int(n), int(t_lo),
          int(t_hi), int(radius), int(patch), float(sigma), float(h), float(alpha), float(beta))
    return out


def estimate_noise(frames: torch.Tensor) -> torch.Tensor:
    """The noise level of each frame in grey levels, Immerkaer's estimator (include/maskflow_b200.h, mfn_noise_sigma):
    sqrt(pi/2) / (18 (W-2) (H-2)) times the exact sum of |I * [[1,-2,1],[-2,4,-2],[1,-2,1]]| over the interior pixels and
    the three channels, floored at NOISE_FLOOR so that it is always positive.  frames (F,H,W,3) or (H,W,3) uint8, H and
    W at least 3.  Returns (F,) float64 on the device (a 0-d tensor for one (H,W,3) frame).  Bit-reproducible.  Sharp
    edges count as noise: on clean, detailed footage the estimate is high."""
    if not isinstance(frames, torch.Tensor) or frames.dim() not in (3, 4):
        raise MaskflowError("estimate_noise: frames must be an (F,H,W,3) or (H,W,3) uint8 tensor")
    fr = frames if frames.dim() == 4 else frames.unsqueeze(0)
    fr = _stab_tensor(fr, "frames", torch.uint8, 3, "estimate_noise")
    F, H, W, _ = fr.shape
    if H < 3 or W < 3:
        raise MaskflowError(f"estimate_noise: frames of {H}x{W} have no interior pixel (H and W must be >= 3)")
    sigma = torch.empty((F,), dtype=torch.float64, device=fr.device)
    _call("mfn_noise_sigma", fr.device, _p(fr), _p(sigma), F, H, W)
    return sigma if frames.dim() == 4 else sigma[0]


def median_noise(frames: torch.Tensor) -> float:
    """The median of estimate_noise over the frames (the lower middle value for an even count), as a float: the sigma
    the video denoisers use when none is given."""
    s = estimate_noise(frames).sort().values
    return float(s[(len(s) - 1) // 2])


# ----------------------------------------------------------------------------------------------------------
# Dense point tracking (csrc/track.cu)
# ----------------------------------------------------------------------------------------------------------
TRACK_EMPTY, TRACK_TRACKED, TRACK_BORN, TRACK_LEFT, TRACK_OCCLUDED, TRACK_BOUNDARY = range(6)


def _finite_nonneg(v) -> bool:
    try:
        return 0.0 <= float(v) < float("inf")
    except (TypeError, ValueError):
        return False


def check_track_args(spacing, queries, who: str) -> torch.Tensor:
    """TrackState's rules for spacing and queries.  Returns the queries as an (M,3) float64 host tensor."""
    if not (isinstance(spacing, int) and not isinstance(spacing, bool) and spacing >= 1):
        raise MaskflowError(f"{who}: spacing must be an integer >= 1, got {spacing!r}")
    q = torch.zeros((0, 3), dtype=torch.float32) if queries is None else torch.as_tensor(queries).detach()
    if q.dim() != 2 or q.shape[1] != 3 or q.dtype.is_complex:
        raise MaskflowError(f"{who}: queries must be (M,3) rows (t, x, y), got {tuple(q.shape)}")
    q = q.to("cpu", torch.float64)
    t = q[:, 0]
    if q.shape[0] and not bool(((t >= 0) & (t < 1 << 24) & (t == torch.floor(t))).all()):
        raise MaskflowError(f"{who}: every query's t must be an integer frame index in [0, 2^24)")
    return q


class TrackState:
    """Device-side state of the dense point tracker (include/maskflow_b200.h, "Dense point tracking") for H x W frames.

    pos (K,2) float32 (x,y) and status (K,) uint8 (TRACK_EMPTY ... TRACK_BOUNDARY) of the slots in the current frame;
    cells (Gy,Gx) uint8, the cells its live tracks cover; frame (1,) int32, the index of the next frame to seed; dropped
    (1,) int32, the candidates of the last seeded frame left without a slot; and the seed kernel's workspace.  Slots
    0..M-1 belong to `queries`, M rows (t, x, y) with t an integer frame index; max_tracks dense slots follow (default
    2 Gx Gy, Gx = W // spacing, Gy = H // spacing).  tau: the texture threshold relative to the frame's largest; alpha,
    beta: the forward-backward check; boundary: (alpha_b, beta_b) of the motion-boundary test.  Everything is allocated
    here once: the track_* ops write into it and allocate nothing else for the state, so a sequence of them can be
    captured in a CUDA graph.  reset() returns it to the start of a video."""

    def __init__(self, H: int, W: int, spacing: int = 8, tau: float = 0.001, alpha: float = 0.01, beta: float = 0.5,
                 boundary=(0.01, 0.002), max_tracks: Optional[int] = None, queries=None, device=None):
        q = check_track_args(spacing, queries, "TrackState")
        if int(H) < 1 or int(W) < 1 or int(H) * int(W) >= 1 << 31:
            raise MaskflowError(f"TrackState: frame size {H}x{W} outside 1 <= H, W and H*W < 2^31")
        try:
            ab, bb = boundary
        except (TypeError, ValueError):
            raise MaskflowError(f"TrackState: boundary must be a pair (alpha_b, beta_b), got {boundary!r}") from None
        for v, nm in ((tau, "tau"), (alpha, "alpha"), (beta, "beta"), (ab, "boundary alpha_b"), (bb, "boundary beta_b")):
            if not _finite_nonneg(v):
                raise MaskflowError(f"TrackState: {nm} must be finite and non-negative, got {v!r}")
        self.H, self.W, self.spacing = int(H), int(W), int(spacing)
        self.Gx, self.Gy = self.W // self.spacing, self.H // self.spacing
        self.tau, self.alpha, self.beta = float(tau), float(alpha), float(beta)
        self.boundary = (float(ab), float(bb))
        self.M = int(q.shape[0])
        dense = 2 * self.Gx * self.Gy if max_tracks is None else max_tracks
        if not (isinstance(dense, int) and not isinstance(dense, bool) and dense >= 0):
            raise MaskflowError(f"TrackState: max_tracks must be a non-negative integer, got {max_tracks!r}")
        self.K = self.M + dense
        if self.K < 1 or self.K >= 1 << 31:
            raise MaskflowError(f"TrackState: {self.K} slots ({self.M} queries, {dense} dense): need 1 <= K < 2^31")
        dev = torch.device("cuda") if device is None else torch.device(device)
        self.pos = torch.empty((self.K, 2), dtype=torch.float32, device=dev)
        self.device = dev = self.pos.device          # with its index: tensors are compared against it
        self.queries = q.to(dev, torch.float32).contiguous()
        self.status = torch.empty((self.K,), dtype=torch.uint8, device=dev)
        self.cells = torch.zeros((self.Gy, self.Gx), dtype=torch.uint8, device=dev)
        self.frame = torch.empty((1,), dtype=torch.int32, device=dev)
        self.dropped = torch.empty((1,), dtype=torch.int32, device=dev)
        self.ws_bytes = int(_lib.lib().mfn_track_seed_workspace_bytes(self.K))
        self.ws = torch.empty((self.ws_bytes,), dtype=torch.uint8, device=dev)
        self.reset()

    def reset(self) -> None:
        """The start of a video: no tracks (NaN positions, EMPTY, no covered cell), frame 0 next."""
        self.pos.fill_(float("nan"))
        self.status.zero_()
        self.cells.zero_()
        self.frame.zero_()
        self.dropped.zero_()


def _track_tensor(t, nm: str, dtype, shape, who: str) -> torch.Tensor:
    if not isinstance(t, torch.Tensor) or not t.is_cuda:
        raise MaskflowError(f"{who}: {nm} must be a CUDA tensor; the hot path has no CPU implementation")
    if t.dtype != dtype or not t.is_contiguous():
        raise MaskflowError(f"{who}: {nm} must be a contiguous {dtype} tensor")
    if tuple(t.shape) != tuple(shape):
        raise MaskflowError(f"{who}: expected {nm} of shape {tuple(shape)}, got {tuple(t.shape)}")
    return t


def track_texture(frames: torch.Tensor, spacing: int = 8):
    """Seed-point texture of uint8 frames (F,H,W,3) (or one (H,W,3) frame), any channel order: the smaller eigenvalue of
    the 5x5 structure tensor of R+G+B at each seed point (i h + h/2, j h + h/2), h = spacing, exact in float64
    (include/maskflow_b200.h, mfn_track_texture).  Returns (lambda2 (F,Gy,Gx) float64, lambda_max (F,) float64, each
    frame's largest); an (H,W,3) frame gives (Gy,Gx) and (1,)."""
    if not isinstance(frames, torch.Tensor) or frames.dim() not in (3, 4):
        raise MaskflowError("track_texture: frames must be an (F,H,W,3) or (H,W,3) uint8 CUDA tensor")
    f4 = frames if frames.dim() == 4 else frames.unsqueeze(0)
    F, H, W = (int(s) for s in f4.shape[:3])
    _track_tensor(f4, "frames", torch.uint8, (F, H, W, 3), "track_texture")
    if not (isinstance(spacing, int) and spacing >= 1):
        raise MaskflowError(f"track_texture: spacing must be an integer >= 1, got {spacing!r}")
    lam = torch.empty((F, H // spacing, W // spacing), dtype=torch.float64, device=f4.device)
    lmax = torch.empty((F,), dtype=torch.float64, device=f4.device)
    _call("mfn_track_texture", f4.device, _p(f4), _p(lam), _p(lmax), F, H, W, int(spacing))
    return (lam, lmax) if frames.dim() == 4 else (lam[0], lmax)


def track_advance(state: TrackState, flow_fw: torch.Tensor, flow_bw: torch.Tensor) -> None:
    """Moves every track of `state` from frame k to k+1 along flow_fw (k -> k+1) and flow_bw (k+1 -> k), (H,W,2) float32
    (x,y) pixels: TRACKED at p + flow_fw(p), or stopped LEFT, OCCLUDED (forward-backward check) or BOUNDARY (flow
    gradient), and marks the cells the tracks cover (include/maskflow_b200.h, mfn_track_advance).  Forward only."""
    shape = (state.H, state.W, 2)
    _track_tensor(flow_fw, "flow_fw", torch.float32, shape, "track_advance")
    _track_tensor(flow_bw, "flow_bw", torch.float32, shape, "track_advance")
    if flow_fw.device != state.device or flow_bw.device != state.device:
        raise MaskflowError(f"track_advance: the flows must be on the state's device {state.device}")
    _no_grad_path("track_advance", flow_fw, flow_bw)
    ab, bb = state.boundary
    _call("mfn_track_advance", state.device, _p(flow_fw), _p(flow_bw), _p(state.pos), _p(state.status), _p(state.cells),
          state.K, state.H, state.W, state.spacing, state.alpha, state.beta, ab, bb)


def track_seed(state: TrackState, lambda2: torch.Tensor, lambda_max: torch.Tensor, out_xy=None, out_status=None,
               out_dropped=None):
    """The births of the frame `state.frame` (on the device): query births, then new tracks at the seed points of the
    uncovered cells with lambda2 > 0 and lambda2 >= tau lambda_max, in row-major cell order, into the free dense slots in
    slot order (include/maskflow_b200.h, mfn_track_seed).  lambda2 (Gy,Gx) and lambda_max (1,) float64 of that frame, as
    track_texture returns them.  Returns the frame's (xy (K,2) float32, status (K,) uint8, dropped (1,) int32), written
    into out_xy, out_status and out_dropped when given (dropped defaults to state.dropped)."""
    _track_tensor(lambda2, "lambda2", torch.float64, (state.Gy, state.Gx), "track_seed")
    _track_tensor(lambda_max, "lambda_max", torch.float64, (1,), "track_seed")
    xy = torch.empty((state.K, 2), dtype=torch.float32, device=state.device) if out_xy is None else out_xy
    st = torch.empty((state.K,), dtype=torch.uint8, device=state.device) if out_status is None else out_status
    dropped = state.dropped if out_dropped is None else out_dropped
    _track_tensor(xy, "out_xy", torch.float32, (state.K, 2), "track_seed")
    _track_tensor(st, "out_status", torch.uint8, (state.K,), "track_seed")
    _track_tensor(dropped, "out_dropped", torch.int32, (1,), "track_seed")
    for t in (lambda2, lambda_max, xy, st, dropped):
        if t.device != state.device:
            raise MaskflowError(f"track_seed: every tensor must be on the state's device {state.device}")
    _call("mfn_track_seed", state.device, _p(lambda2), _p(lambda_max), _p(state.queries) if state.M else None, state.M,
          _p(state.pos), _p(state.status), _p(state.cells), _p(state.frame), _p(dropped), _p(state.ws), state.ws_bytes,
          _p(xy), _p(st), state.K, state.H, state.W, state.spacing, state.tau)
    return xy, st, dropped


def track_start(state: TrackState, frame: torch.Tensor, out_xy=None, out_status=None, out_dropped=None):
    """Frame 0 of a video: state.reset(), then the seeds (and the queries born) in `frame` (H,W,3) uint8.  Returns
    track_seed's (xy, status, dropped)."""
    state.reset()
    lam, lmax = track_texture(frame, state.spacing)
    return track_seed(state, lam, lmax, out_xy, out_status, out_dropped)


def track_step(state: TrackState, flow_fw: torch.Tensor, flow_bw: torch.Tensor, frame: torch.Tensor, out_xy=None,
               out_status=None, out_dropped=None):
    """One frame k -> k+1: track_advance along the pair's flows, then track_seed in frame k+1 (H,W,3) uint8.  Returns
    track_seed's (xy, status, dropped)."""
    track_advance(state, flow_fw, flow_bw)
    lam, lmax = track_texture(frame, state.spacing)
    return track_seed(state, lam, lmax, out_xy, out_status, out_dropped)


# ----------------------------------------------------------------------------------------------------------
# Unsupervised losses (csrc/unsup_loss.cu): census photometric loss and second-order smoothness
# ----------------------------------------------------------------------------------------------------------
def unsup_workspace_bytes(loss: str, N: int, H: int, W: int) -> int:
    """Bytes of the `ws` scratch of mfn_census_loss_forward ("census") / mfn_smoothness_loss_forward ("smoothness")
    (include/maskflow_b200.h, "Unsupervised losses")."""
    if loss == "census":
        return 8 * N * (-(-H // 8)) * (-(-W // 32))
    if loss == "smoothness":
        return 8 * N * (-(-H * W // 256))
    raise MaskflowError(f"unsup_workspace_bytes: unknown loss {loss!r}")


def _census_forward(img1, img2w, occ):
    """(loss (N,), vsum (N,), coef (N,H,W)) of mfn_census_loss_forward."""
    N, _, H, W = img1.shape
    dev = img1.device
    loss = torch.empty(N, device=dev, dtype=torch.float32)
    vsum = torch.empty(N, device=dev, dtype=torch.float32)
    coef = torch.empty((N, H, W), device=dev, dtype=torch.float32)
    nb = unsup_workspace_bytes("census", N, H, W)
    ws = torch.empty(nb // 4, device=dev, dtype=torch.float32)
    _call("mfn_census_loss_forward", dev, _p(img1), _p(img2w), _p(occ), _p(coef), _p(vsum), _p(loss), _p(ws), nb, N, H, W)
    return loss, vsum, coef


def _census_backward(img1, img2w, coef, vsum, g):
    N, _, H, W = img1.shape
    gi = torch.empty_like(img2w)
    _call("mfn_census_loss_backward", img1.device, _p(img1), _p(img2w), _p(coef), _p(vsum), _p(g), _p(gi), N, H, W)
    return gi


def _smoothness_forward(flow, img):
    N, _, H, W = flow.shape
    loss = torch.empty(N, device=flow.device, dtype=torch.float32)
    nb = unsup_workspace_bytes("smoothness", N, H, W)
    ws = torch.empty(nb // 4, device=flow.device, dtype=torch.float32)
    _call("mfn_smoothness_loss_forward", flow.device, _p(flow), _p(img), _p(loss), _p(ws), nb, N, H, W)
    return loss


def _smoothness_backward(flow, img, g):
    N, _, H, W = flow.shape
    gf = torch.empty_like(flow)
    _call("mfn_smoothness_loss_backward", flow.device, _p(flow), _p(img), _p(g), _p(gf), N, H, W)
    return gf


class CensusLossFn(torch.autograd.Function):
    """mfn_census_loss_forward / _backward: per-sample census loss (N,) of (img1, img2_warped, occ); the gradient
    reaches img2_warped only (img1 and occ are data).  Inputs are checked by losses.census_loss."""

    @staticmethod
    def forward(ctx, img1, img2w, occ):
        loss, vsum, coef = _census_forward(img1, img2w, occ)
        ctx.save_for_backward(img1, img2w, coef, vsum)
        return loss

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, g):
        img1, img2w, coef, vsum = ctx.saved_tensors
        return None, _census_backward(img1, img2w, coef, vsum, g.contiguous().float()), None


class SmoothnessLossFn(torch.autograd.Function):
    """mfn_smoothness_loss_forward / _backward: per-sample smoothness (N,) of flow weighted by the edges of img; the
    gradient reaches the flow only.  Inputs are checked by losses.smoothness_loss."""

    @staticmethod
    def forward(ctx, flow, img):
        ctx.save_for_backward(flow, img)
        return _smoothness_forward(flow, img)

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, g):
        flow, img = ctx.saved_tensors
        return _smoothness_backward(flow, img, g.contiguous().float()), None
