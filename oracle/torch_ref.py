"""Differentiable torch restatement of the hot-path operators.  TEST INFRASTRUCTURE ONLY.

Same semantics as oracle/mfn_oracle.c (which it is checked against in tests/test_oracle.py), written as
plain torch expressions so that torch.autograd yields the analytic backward used to check the CUDA
backward kernels.  Only tests/, __graft_entry__.smoke() and bench.py's reference legs may import it.

Reference call sites (all in /root/reference):
  correlation         network/MaskFlownet.py:193-195, 440-441   (F.Correlation)
  deformable_conv     network/layer.py:117-124                   (F.contrib.DeformableConvolution)
  upsample            network/MaskFlownet.py:35-62               (Upsample block)
  reconstruction2d    network/layer.py:8-18                      (GridGenerator('warp') + BilinearSampler)
  warp_mask           network/MaskFlownet.py:227-233             (one pyramid level of the S head)
  image_warp_concat   network/MaskFlownet.py:308-313             (cascade input)
"""
from __future__ import annotations

import torch
import torch.nn.functional as tF


def correlation(f1: torch.Tensor, f2: torch.Tensor, max_displacement: int = 4) -> torch.Tensor:
    """out[n,(dy+md)*(2md+1)+(dx+md),y,x] = mean_c f1[n,c,y,x] * f2[n,c,y+dy,x+dx], zero outside.

    Regime used by the reference: pad_size = max_displacement, kernel_size = 1, strides 1, multiply."""
    md = max_displacement
    N, C, H, W = f1.shape
    f2p = tF.pad(f2, (md, md, md, md))
    planes = []
    for dy in range(-md, md + 1):
        for dx in range(-md, md + 1):
            shifted = f2p[:, :, md + dy:md + dy + H, md + dx:md + dx + W]
            planes.append((f1 * shifted).sum(dim=1) / C)
    return torch.stack(planes, dim=1)


def _gather_plane(x: torch.Tensor, hi: torch.Tensor, wi: torch.Tensor) -> torch.Tensor:
    """x (N,C,H,W); integer index maps hi, wi (N,OH,OW), already inside the image -> (N,C,OH,OW)."""
    N, C, H, W = x.shape
    OH, OW = hi.shape[1:]
    idx = (hi * W + wi).view(N, 1, OH * OW).expand(N, C, OH * OW)
    return x.reshape(N, C, H * W).gather(2, idx).view(N, C, OH, OW)


def sample_tap(x: torch.Tensor, h: torch.Tensor, w: torch.Tensor, border_mode: int = 0) -> torch.Tensor:
    """Bilinear sample of x (N,C,H,W) at real positions h, w (N,OH,OW).

    border_mode 0: MXNet-1.5 deformable_im2col rule (zero unless 0<=h<H and 0<=w<W; a coordinate whose
    floor is >= size-1 collapses onto the last row/column).  border_mode 1: zero-corner (DCNv2) rule."""
    N, C, H, W = x.shape
    h0 = torch.floor(h)
    w0 = torch.floor(w)
    if border_mode == 0:
        inside = (h >= 0) & (w >= 0) & (h < H) & (w < W)
        ch = h0 >= H - 1
        cw = w0 >= W - 1
        lh = torch.where(ch, torch.zeros_like(h), h - h0)
        lw = torch.where(cw, torch.zeros_like(w), w - w0)
        h0i = torch.where(ch, torch.full_like(h0, H - 1), h0).clamp(0, H - 1).long()
        w0i = torch.where(cw, torch.full_like(w0, W - 1), w0).clamp(0, W - 1).long()
        h1i = torch.where(ch, h0i, (h0i + 1).clamp(max=H - 1))
        w1i = torch.where(cw, w0i, (w0i + 1).clamp(max=W - 1))
        hh, hw = 1 - lh, 1 - lw
        val = ((hh * hw).unsqueeze(1) * _gather_plane(x, h0i, w0i)
               + (hh * lw).unsqueeze(1) * _gather_plane(x, h0i, w1i)
               + (lh * hw).unsqueeze(1) * _gather_plane(x, h1i, w0i)
               + (lh * lw).unsqueeze(1) * _gather_plane(x, h1i, w1i))
        return val * inside.unsqueeze(1).to(val.dtype)
    inside = (h > -1) & (w > -1) & (h < H) & (w < W)
    lh, lw = h - h0, w - w0
    hh, hw = 1 - lh, 1 - lw
    h0i, w0i = h0.long(), w0.long()
    h1i, w1i = h0i + 1, w0i + 1
    val = 0
    for (hi, wi, wt) in ((h0i, w0i, hh * hw), (h0i, w1i, hh * lw), (h1i, w0i, lh * hw), (h1i, w1i, lh * lw)):
        ok = (hi >= 0) & (hi <= H - 1) & (wi >= 0) & (wi <= W - 1) & inside
        v = _gather_plane(x, hi.clamp(0, H - 1), wi.clamp(0, W - 1))
        val = val + (wt * ok.to(wt.dtype)).unsqueeze(1) * v
    return val


def deformable_conv(x, offset, weight, bias=None, border_mode: int = 0):
    """3x3 / stride 1 / pad 1 / dilation 1 / one group deformable convolution (the reference's kwargs,
    network/layer.py:91-95).  offset (N,18,H,W): channel 2k = dy, 2k+1 = dx of tap k = i*3+j."""
    N, C, H, W = x.shape
    Fo = weight.shape[0]
    assert weight.shape[1:] == (C, 3, 3) and offset.shape == (N, 18, H, W)
    ys = torch.arange(H, dtype=x.dtype, device=x.device).view(1, H, 1)
    xs = torch.arange(W, dtype=x.dtype, device=x.device).view(1, 1, W)
    cols = []
    for i in range(3):
        for j in range(3):
            k = i * 3 + j
            h = (ys + (i - 1)) + offset[:, 2 * k]
            w = (xs + (j - 1)) + offset[:, 2 * k + 1]
            cols.append(sample_tap(x, h, w, border_mode))
    col = torch.stack(cols, dim=2)  # N, C, 9, H, W
    out = torch.einsum("fck,nckhw->nfhw", weight.reshape(Fo, C, 9), col)
    if bias is not None:
        out = out + bias.view(1, Fo, 1, 1)
    return out


def upsample(x: torch.Tensor, factor: int) -> torch.Tensor:
    """Reference Upsample(f): edge-pad bottom/right by one, fixed-kernel transposed conv, crop."""
    if factor == 1:
        return x
    N, C, H, W = x.shape
    f = factor
    c = f - 1
    t = torch.arange(2 * f - 1, dtype=x.dtype, device=x.device)
    k1 = 1 - (c - t).abs() / (c + 1)
    k2 = (k1[:, None] * k1[None, :]).view(1, 1, 2 * f - 1, 2 * f - 1)
    b = x.reshape(N * C, 1, H, W)
    b = tF.pad(b, (0, 1, 0, 1), mode="replicate")
    up = tF.conv_transpose2d(b, k2, stride=f, padding=f - 1)
    return up[:, :, :-1, :-1].reshape(N, C, f * H, f * W)


def reconstruction2d(x: torch.Tensor, flow_yx: torch.Tensor) -> torch.Tensor:
    """layer.Reconstruction2D: sample x at (y + flow[:,0], x + flow[:,1]), zero outside."""
    N, C, H, W = x.shape
    ys = torch.arange(H, dtype=x.dtype, device=x.device).view(1, H, 1)
    xs = torch.arange(W, dtype=x.dtype, device=x.device).view(1, 1, W)
    gx = (flow_yx[:, 1] + xs) / ((W - 1) / 2) - 1
    gy = (flow_yx[:, 0] + ys) / ((H - 1) / 2) - 1
    grid = torch.stack([gx, gy], dim=-1)
    return tF.grid_sample(x, grid, mode="bilinear", padding_mode="zeros", align_corners=True)


def leaky(x, slope=0.1):
    return tF.leaky_relu(x, slope)


def warp_mask(x, flow_coarse, mask_coarse, weight, bias, tradeoff, scale: float, stride: int,
              upsample_factor: int = 2, border_mode: int = 0, slope: float = 0.1):
    """One S-head level, network/MaskFlownet.py:228-233 (level 5; same at :246-251, :264-269, :282-287):
        flow = Upsample(2)(flow_c); mask = Upsample(2)(mask_c)
        warp = deform(x, repeat(flow*scale/stride, 9)); warp = warp*sigmoid(mask) + tradeoff; LeakyReLU
    mask_coarse / tradeoff may be None (cascade variant, MaskFlownet.py:465-466: LeakyReLU only).
    Returns (warp, flow_up, mask_up)."""
    flow = upsample(flow_coarse, upsample_factor)
    mask = upsample(mask_coarse, upsample_factor) if mask_coarse is not None else None
    off = (flow * scale / stride).unsqueeze(1).repeat(1, 9, 1, 1, 1).reshape(flow.shape[0], 18, *flow.shape[2:])
    warp = deformable_conv(x, off, weight, bias, border_mode)
    if mask is not None:
        warp = warp * torch.sigmoid(mask)
    if tradeoff is not None:
        warp = warp + tradeoff
    return leaky(warp, slope), flow, mask


def image_warp_concat(im2, flow2, mask2, scale: float):
    """network/MaskFlownet.py:308-313: c40 = [warp(im2, Upsample(4)(flow2)*scale) ; sigmoid(Upsample(4)(mask2)) - 0.5]."""
    mask0 = torch.sigmoid(upsample(mask2, 4)) - 0.5
    warped = reconstruction2d(im2, upsample(flow2, 4) * scale)
    return torch.cat([warped, mask0], dim=1)
