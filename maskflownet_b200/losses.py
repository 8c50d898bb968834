"""Training losses of the reference (network/MaskFlownet.py:548-611), on the CUDA Upsample operator.

EpeLossWithMask: per-sample  sum_hw( sqrt(sum_c (pred-label)^2 + eps) * mask ) / sum_hw(mask)     (q-robust variant:
(sum_c |pred-label| + eps)^q).  MultiscaleEpe('upsampling'): sum_i w_i * EpeLossWithMask(Upsample(s_i)(pred_i), flow, mask)
with s = [64, 32, 16, 8, 4] and w = [.005, .01, .02, .08, .32] (network/pipeline.py:39-45).  It is what drives the backward
kernels in BASELINE configs[2] and [4].

`multiscale_epe` on CUDA tensors runs the FUSED kernels of csrc/loss.cu (SURVEY.md 8f row N2): one pass over the label and
the mask for all five scales, no up-sampled prediction is materialised, the backward is one gather launch (the composition
of operators below needs ~45 launches forward and, through Upsample(64)'s backward, a 128x128 serial gather per coarse
pixel).  `fused=False` (or a custom `upsample=`) runs the operator-by-operator composition -- the reference's own structure,
kept for A/B runs and used on CPU tensors by the tests' oracle leg.
"""
from __future__ import annotations

import ctypes
from typing import NamedTuple, Optional, Sequence

import torch

from . import _lib, ops
from ._lib import MaskflowError

SCALES = (64, 32, 16, 8, 4)
WEIGHTS = (.005, .01, .02, .08, .32)


def epe_loss_with_mask(pred, label, mask, eps: float = 1e-8, q: Optional[float] = None):
    if q is not None:
        loss = ((pred - label).abs().sum(dim=1) + eps) ** q
    else:
        loss = torch.sqrt((pred - label).square().sum(dim=1) + eps)
    loss = loss * mask.squeeze(1)
    return loss.flatten(1).sum(dim=1) / mask.flatten(1).sum(dim=1)


def _host_arrays(tensors, scales, weights):
    n = len(tensors)
    return ((ctypes.c_void_p * n)(*[t.data_ptr() for t in tensors]), (ctypes.c_int * n)(*[int(s) for s in scales]),
            (ctypes.c_float * n)(*[float(w) for w in weights]))


class _MultiscaleEpeFn(torch.autograd.Function):
    """mfn_multiscale_epe_forward / _backward (csrc/loss.cu); gradients flow to the predictions only (label and mask are data)."""

    @staticmethod
    def forward(ctx, flow, mask, scales, weights, eps, q, *preds):
        N, _, H, W = flow.shape
        dev = flow.device
        pa, sa, wa = _host_arrays(preds, scales, weights)
        loss = torch.empty(N, device=dev, dtype=torch.float32)
        msum = torch.empty(N, device=dev, dtype=torch.float32)
        wsb = int(_lib.lib().mfn_multiscale_epe_workspace_bytes(N))
        ws = torch.empty(wsb // 4, device=dev, dtype=torch.float32)
        ops._call("mfn_multiscale_epe_forward", dev, ops._p(flow), ops._p(mask), pa, sa, wa, len(preds), float(eps), float(q),
                  ops._p(loss), ops._p(msum), ops._p(ws), wsb, N, H, W)
        ctx.cfg = (tuple(scales), tuple(weights), float(eps), float(q))
        ctx.save_for_backward(flow, mask, msum, *preds)
        return loss

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, g):
        flow, mask, msum, *preds = ctx.saved_tensors
        scales, weights, eps, q = ctx.cfg
        N, _, H, W = flow.shape
        grads = [torch.empty_like(p) for p in preds]
        pa, sa, wa = _host_arrays(preds, scales, weights)
        ga = (ctypes.c_void_p * len(grads))(*[t.data_ptr() for t in grads])
        g = g.contiguous().float()
        ops._call("mfn_multiscale_epe_backward", flow.device, ops._p(flow), ops._p(mask), pa, sa, wa, len(preds), eps, q,
                  ops._p(g), ops._p(msum), ga, N, H, W)
        return (None, None, None, None, None, None, *grads)


def multiscale_epe_fused(flow, mask, predictions: Sequence[torch.Tensor], scales=SCALES, weights=WEIGHTS, eps: float = 1e-8,
                         q: Optional[float] = None) -> torch.Tensor:
    """The fused MultiscaleEpe('upsampling'): CUDA float32 tensors only (no fallback).  Returns the per-sample losses (N,)."""
    flow, mask = ops._chk(flow, "multiscale_epe.flow"), ops._chk(mask, "multiscale_epe.mask")
    preds = [ops._chk(p, "multiscale_epe.prediction") for p in predictions]
    N, C, H, W = flow.shape
    if C != 2 or tuple(mask.shape) != (N, 1, H, W):
        raise MaskflowError(f"multiscale_epe: flow must be (N,2,H,W) and mask (N,1,H,W); got {tuple(flow.shape)}, {tuple(mask.shape)}")
    if not (len(preds) == len(scales) == len(weights)):
        raise MaskflowError("multiscale_epe: one scale and one weight per prediction")
    for p, s in zip(preds, scales):
        if H % s or W % s or tuple(p.shape) != (N, 2, H // s, W // s):
            raise MaskflowError(f"multiscale_epe: prediction {tuple(p.shape)} x{s} does not up-sample to the label {tuple(flow.shape)}")
    if flow.requires_grad or mask.requires_grad:
        raise MaskflowError("multiscale_epe: the label and the mask are data (no gradient is computed for them)")
    return _MultiscaleEpeFn.apply(flow, mask, tuple(scales), tuple(weights), eps, -1.0 if q is None else float(q), *preds)


def multiscale_epe(flow, mask, predictions: Sequence[torch.Tensor], scales=SCALES, weights=WEIGHTS, eps: float = 1e-8,
                   q: Optional[float] = None, upsample=None, fused: Optional[bool] = None):
    """flow (N,2,H,W) ground truth in (y,x) order, mask (N,1,H,W); returns the per-sample loss vector (N,).
    CUDA tensors take the fused kernels unless fused=False or a custom `upsample` is given."""
    if fused is None:
        fused = upsample is None and flow.is_cuda
    if fused:
        return multiscale_epe_fused(flow, mask, predictions, scales, weights, eps, q)
    upsample = ops.upsample if upsample is None else upsample
    total = 0
    for p, w, s in zip(predictions, weights, scales):
        total = total + w * epe_loss_with_mask(upsample(p, s), flow, mask, eps, q)
    return total


# ----------------------------------------------------------------------------------------------------------
# Unsupervised fine-tuning on unlabelled pairs (UnFlow, Meister, Hur and Roth, AAAI 2018): csrc/unsup_loss.cu
# ----------------------------------------------------------------------------------------------------------
OCC_ALPHA, OCC_BETA = 0.01, 0.5          # the forward-backward check's constants (Sundaram et al. 2010)


def _unsup_input(t, name: str, channels: Optional[int], dtype=torch.float32, data: bool = True) -> torch.Tensor:
    if not isinstance(t, torch.Tensor) or not t.is_cuda:
        raise MaskflowError(f"{name} must be a CUDA tensor; the hot path has no CPU implementation")
    if t.dtype != dtype or not t.is_contiguous():
        raise MaskflowError(f"{name} must be a contiguous {dtype} tensor, got {t.dtype}"
                            + ("" if t.is_contiguous() else " (non-contiguous)"))
    if t.dim() != (3 if channels is None else 4) or (channels is not None and t.shape[1] != channels):
        raise MaskflowError(f"{name}: expected " + ("(N,H,W)" if channels is None else f"(N,{channels},H,W)")
                            + f", got {tuple(t.shape)}")
    if data and t.requires_grad:
        raise MaskflowError(f"{name} is data: no gradient is computed for it (detach it)")
    return t


def census_loss(img1, img2_warped, occ) -> torch.Tensor:
    """Per-sample occlusion-masked census loss (N,) of img1 against img2_warped, both (N,3,H,W) float32 RGB in [0,1];
    occ (N,H,W) uint8, nonzero = occluded (left out).  The formula is in include/maskflow_b200.h; the gradient reaches
    img2_warped only."""
    img1 = _unsup_input(img1, "census_loss.img1", 3)
    img2_warped = _unsup_input(img2_warped, "census_loss.img2_warped", 3, data=False)
    occ = _unsup_input(occ, "census_loss.occ", None, torch.uint8)
    N, _, H, W = img1.shape
    if img2_warped.shape != img1.shape or tuple(occ.shape) != (N, H, W) or img2_warped.device != img1.device \
            or occ.device != img1.device:
        raise MaskflowError(f"census_loss: shapes differ: img1 {tuple(img1.shape)}, img2_warped "
                            f"{tuple(img2_warped.shape)}, occ {tuple(occ.shape)}")
    if ops._needs_grad(img2_warped):
        return ops.CensusLossFn.apply(img1, img2_warped, occ)
    return ops._census_forward(img1, img2_warped, occ)[0]


def smoothness_loss(flow, img) -> torch.Tensor:
    """Per-sample second-order, edge-aware smoothness (N,) of flow (N,2,H,W) float32 weighted by the edges of img
    (N,3,H,W); the gradient reaches the flow only."""
    flow = _unsup_input(flow, "smoothness_loss.flow", 2, data=False)
    img = _unsup_input(img, "smoothness_loss.img", 3)
    if img.shape[0] != flow.shape[0] or img.shape[2:] != flow.shape[2:] or img.device != flow.device:
        raise MaskflowError(f"smoothness_loss: shapes differ: flow {tuple(flow.shape)}, img {tuple(img.shape)}")
    if ops._needs_grad(flow):
        return ops.SmoothnessLossFn.apply(flow, img)
    return ops._smoothness_forward(flow, img)


class UnsupervisedLoss(NamedTuple):
    loss: torch.Tensor          # (2N,) per-sample photo + smooth_weight * smooth: [a -> b; b -> a]
    occluded: torch.Tensor      # (2N,) share of each sample's pixels the forward-backward check left out
    photo: torch.Tensor         # (2N,) census term
    smooth: torch.Tensor        # (2N,) smoothness term (unweighted)


def unsupervised_loss(a, b, F_fw, F_bw, smooth_weight: float) -> UnsupervisedLoss:
    """The unsupervised loss of a batch of pairs.  a, b (N,3,H,W) float32 in [0,1] (before any colour augmentation or
    centralisation); F_fw, F_bw (N,2,H,W) full-resolution flows a -> b and b -> a in the network's (y,x) order, pixels.
      1. occlusion: ops.flow_consistency on the detached flows (alpha 0.01, beta 0.5), no gradient;
      2. warp: b~ = reconstruction2d(b, F_fw), a~ = reconstruction2d(a, F_bw) (the gradient reaches the flows);
      3. census on (a, b~, occ_fw) and (b, a~, occ_bw), batched as 2N;
      4. smoothness of F_fw with the edges of a and of F_bw with the edges of b;
      5. loss = census + smooth_weight * smoothness per sample."""
    a = _unsup_input(a, "unsupervised_loss.a", 3)
    b = _unsup_input(b, "unsupervised_loss.b", 3)
    for t, nm in ((F_fw, "F_fw"), (F_bw, "F_bw")):
        if not isinstance(t, torch.Tensor) or t.shape != (a.shape[0], 2) + tuple(a.shape[2:]):
            raise MaskflowError(f"unsupervised_loss: {nm} must be (N,2,H,W) like the images, got "
                                f"{tuple(getattr(t, 'shape', ()))}")
    if b.shape != a.shape:
        raise MaskflowError(f"unsupervised_loss: a {tuple(a.shape)} and b {tuple(b.shape)} differ")
    with torch.no_grad():
        xy = lambda f: f.detach().flip(1).permute(0, 2, 3, 1).contiguous()  # noqa: E731
        occ = torch.cat(ops.flow_consistency(xy(F_fw), xy(F_bw), OCC_ALPHA, OCC_BETA))
    warped = torch.cat([ops.reconstruction2d(b, F_fw), ops.reconstruction2d(a, F_bw)])
    images = torch.cat([a, b])
    photo = census_loss(images, warped, occ)
    smooth = smoothness_loss(torch.cat([F_fw, F_bw]), images)
    return UnsupervisedLoss(photo + smooth_weight * smooth, occ.flatten(1).float().mean(1), photo, smooth)
