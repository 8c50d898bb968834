"""float64, differentiable torch restatement of the unsupervised losses (csrc/unsup_loss.cu, include/maskflow_b200.h,
"Unsupervised losses"), written from their formulas; its autograd is the checker of the backward kernels.

    census_loss(img1, img2w, occ)     -> per-sample photometric loss and what it is built from (d, v, coef, vsum)
    smoothness_loss(flow, img)        -> per-sample second-order, edge-aware smoothness
    occlusion(F_fw, F_bw)             -> the forward-backward check (Sundaram et al. 2010) on (y,x) flows, float64
    unsupervised_loss(a, b, F_fw, F_bw, smooth_weight, occ=None)
                                      -> the composition: occlusion, warp (torch_ref.reconstruction2d), census on both
                                         directions batched as 2N, smoothness with the edges of each direction's image 1

Images (N,3,H,W) in [0,1]; flows (N,2,H,W) in the network's (y,x) order, pixels.  Everything is computed in the dtype of
the inputs (the tests pass float64).  `offsets` exists for the tests' controls (a dropped census offset).
"""
from __future__ import annotations

import torch
import torch.nn.functional as tF

from . import torch_ref

R = 3
OFFSETS = tuple((dy, dx) for dy in range(-R, R + 1) for dx in range(-R, R + 1) if (dy, dx) != (0, 0))
GREY = (0.2989, 0.5870, 0.1140)
EPS_RHO, P_RHO = 1e-6, 0.45


def grey(img: torch.Tensor) -> torch.Tensor:
    return 255.0 * (GREY[0] * img[:, 0] + GREY[1] * img[:, 1] + GREY[2] * img[:, 2])


def census_t(delta: torch.Tensor) -> torch.Tensor:
    return delta / torch.sqrt(0.81 + delta * delta)


def interior(H: int, W: int, device=None) -> torch.Tensor:
    m = torch.zeros(H, W, dtype=torch.bool, device=device)
    m[R:H - R, R:W - R] = True
    return m


def census_distance(img1, img2w, offsets=OFFSETS) -> torch.Tensor:
    """d (N,H,W) on the interior pixels, 0 elsewhere."""
    g1, g2 = grey(img1), grey(img2w)
    N, H, W = g1.shape
    if H < 2 * R + 1 or W < 2 * R + 1:
        return torch.zeros_like(g1)
    c1, c2 = g1[:, R:H - R, R:W - R], g2[:, R:H - R, R:W - R]
    d = torch.zeros_like(c1)
    for dy, dx in offsets:
        n1 = g1[:, R + dy:H - R + dy, R + dx:W - R + dx]
        n2 = g2[:, R + dy:H - R + dy, R + dx:W - R + dx]
        s = census_t(n1 - c1) - census_t(n2 - c2)
        d = d + s * s / (0.1 + s * s)
    return tF.pad(d, (R, R, R, R))


def rho(d):
    return (d * d + EPS_RHO) ** P_RHO


def rho_prime(d):
    return 2.0 * P_RHO * d * (d * d + EPS_RHO) ** (P_RHO - 1.0)


def census_loss(img1, img2w, occ, offsets=OFFSETS):
    """(loss (N,), d (N,H,W), v (N,H,W), coef = v rho'(d) (N,H,W), vsum (N,)); occ nonzero = occluded."""
    N, _, H, W = img1.shape
    d = census_distance(img1, img2w, offsets)
    v = (occ == 0).to(d.dtype) * interior(H, W, d.device).to(d.dtype)
    vsum = v.flatten(1).sum(1)
    loss = (v * rho(d)).flatten(1).sum(1) / vsum.clamp(min=1.0)
    return loss, d, v, v * rho_prime(d), vsum


def _edge_weight(diff):
    """exp(-10 (1/3) sum_k |diff_k| / 2) of a channel difference (N,3,...)."""
    return torch.exp(-10.0 * diff.abs().mean(dim=1) / 2.0)


def smoothness_loss(flow, img) -> torch.Tensor:
    N, _, H, W = flow.shape
    loss = flow.new_zeros(N)
    if W > 2:
        wx = _edge_weight(img[..., 2:] - img[..., :-2])
        d2x = flow[..., :-2] - 2.0 * flow[..., 1:-1] + flow[..., 2:]
        loss = loss + (wx[:, None] * d2x.abs()).flatten(1).sum(1) / (2 * H * (W - 2))
    if H > 2:
        wy = _edge_weight(img[:, :, 2:] - img[:, :, :-2])
        d2y = flow[:, :, :-2] - 2.0 * flow[:, :, 1:-1] + flow[:, :, 2:]
        loss = loss + (wy[:, None] * d2y.abs()).flatten(1).sum(1) / (2 * (H - 2) * W)
    return loss


def occlusion(F_fw, F_bw, alpha: float = 0.01, beta: float = 0.5):
    """(occ_fw, occ_bw) bool (N,H,W): a pixel whose target leaves [0, W-1] x [0, H-1], or whose flow and the other
    direction's flow sampled bilinearly at the target fail |w + w'|^2 <= alpha (|w|^2 + |w'|^2) + beta.  No gradient."""
    def one(f, g):
        N, _, H, W = f.shape
        ys = torch.arange(H, dtype=f.dtype, device=f.device).view(1, H, 1)
        xs = torch.arange(W, dtype=f.dtype, device=f.device).view(1, 1, W)
        qy, qx = ys + f[:, 0], xs + f[:, 1]
        inside = (qx >= 0) & (qx <= W - 1) & (qy >= 0) & (qy <= H - 1)
        gs = torch_ref.reconstruction2d(g, f)      # bilinear inside the frame: the same corners as the clamped rule
        d2 = ((f + gs) ** 2).sum(1)
        rhs = alpha * ((f ** 2).sum(1) + (gs ** 2).sum(1)) + beta
        return ~inside | ~(d2 <= rhs)
    with torch.no_grad():
        return one(F_fw, F_bw), one(F_bw, F_fw)


def unsupervised_loss(a, b, F_fw, F_bw, smooth_weight: float, occ=None, warp=torch_ref.reconstruction2d):
    """Per-sample losses (2N,) = census + smooth_weight * smoothness over [a->b; b->a], and (photo, smooth, occ_fw,
    occ_bw).  occ: given (occ_fw, occ_bw), or None for occlusion(F_fw, F_bw)."""
    occ_fw, occ_bw = occlusion(F_fw, F_bw) if occ is None else occ
    b_w, a_w = warp(b, F_fw), warp(a, F_bw)
    photo = census_loss(torch.cat([a, b]), torch.cat([b_w, a_w]), torch.cat([occ_fw, occ_bw]).to(torch.uint8))[0]
    smooth = smoothness_loss(torch.cat([F_fw, F_bw]), torch.cat([a, b]))
    return photo + smooth_weight * smooth, (photo, smooth, occ_fw, occ_bw)
