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


def conv3x3_slices(buf_in: torch.Tensor, c_in0: int, Cin: int, packed: torch.Tensor, bias: Optional[torch.Tensor],
                   buf_out: torch.Tensor, c_out0: int, Cout: int, leaky_slope: float = 0.1, dilation: int = 1,
                   stride: int = 1, depth_to_space: bool = False, linear_prefix: int = 0) -> None:
    """out = LeakyReLU(conv3x3(buf_in[:, c_in0:c_in0+Cin]) + bias) written to buf_out[:, c_out0:c_out0+Cout]; both buffers
    dense NCHW (they may be the same tensor: the dense block's concat buffer).  stride 2 (pad 1) = the pyramid's
    down-sampling convolutions: buf_out is then ((H-1)//2+1, (W-1)//2+1).  depth_to_space: the Cout = 4F conv channels
    are written as F channels of a (2H, 2W) image (sub-pixel phases; see conv_transpose4x4_pack).  linear_prefix: the first
    k output channels skip the activation (MFN_CONV_OUT_LINEAR_PREFIX).  Inference only."""
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
          Cout, int(stride), int(dilation), (1 if depth_to_space else 0) | (int(linear_prefix) << 8), float(leaky_slope),
          _p(ws), ws_bytes)


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
            dilation: int = 1, stride: int = 1):
    """3x3 convolution, padding = dilation, stride 1 (decoder / context network) or 2 (pyramid), + LeakyReLU."""
    x = _chk(x, "conv3x3.x")
    out = torch.empty((x.shape[0], Cout, (x.shape[2] - 1) // stride + 1, (x.shape[3] - 1) // stride + 1), device=x.device,
                      dtype=torch.float32)
    conv3x3_slices(x, 0, x.shape[1], packed, bias, out, 0, Cout, leaky_slope, dilation, stride)
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
    the network (network/pipeline.py:206-212, 85-87, 117-130).  Returns (im1, im2, rgb_mean (N,C,1,1)).  Forward only."""
    for t, nm in ((img1, "img1"), (img2, "img2")):
        if not (t.is_cuda and t.is_contiguous() and t.dim() == 4 and t.dtype in (torch.uint8, torch.float32)):
            raise MaskflowError(f"preprocess: {nm} must be a contiguous CUDA uint8 / float32 NCHW tensor")
    if img1.shape != img2.shape or img1.dtype != img2.dtype:
        raise MaskflowError("preprocess: img1 and img2 must agree in shape and dtype")
    _no_grad_path("preprocess", img1, img2)
    N, C, H, W = img1.shape
    OH, OW = (H, W) if out_hw is None else (int(out_hw[0]), int(out_hw[1]))
    o1 = torch.empty((N, C, OH, OW), device=img1.device, dtype=torch.float32)
    o2 = torch.empty_like(o1)
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
