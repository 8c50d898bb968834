"""float64 numpy restatement of video denoising (csrc/denoise.cu; the rules are in include/maskflow_b200.h, "Video
denoising"), written from the rules.

    denoise(frames, flow_fw, flow_bw, radius, sigma, h, patch, alpha, beta, t0, n, t_lo, t_hi)
                                  -> (n,H,W,3) uint8: the ring form of mfn_denoise_frames
    noise_sums(frames)            -> (F,) int64: S, the sum of |Laplacian-difference filter| over channels and interior
    noise_sigma(frames)           -> (F,) float64: mfn_noise_sigma, bit-identical to the kernel (the same float64
                                     expression of the same exact integer)

Positions are float32, as the rule defines them: q = q_{k-1} + float32(w), w the bilinear sample at q_{k-1} in
float64, so the oracle's chain state has the kernel's type.  The samples, the round-trip test, the colours, the patch
distances and the weights are float64.  h may be inf: every defined neighbour then gets weight 1 (plain averaging along
the flow), the tests' control.
"""
from __future__ import annotations

import numpy as np

NOISE_FLOOR = 0.5
SQRT_HALF_PI = 1.2533141373155003


def _sample(plane, qx, qy):
    """(n,C) float64 bilinear samples of the (H,W,C) plane at positions inside the frame, the kernel's corner rule."""
    H, W = plane.shape[:2]
    x0, y0 = np.floor(qx).astype(np.int64), np.floor(qy).astype(np.int64)
    x1, y1 = np.minimum(x0 + 1, W - 1), np.minimum(y0 + 1, H - 1)
    wx, wy = (qx - x0)[:, None], (qy - y0)[:, None]
    g = plane.astype(np.float64)
    with np.errstate(invalid="ignore"):                # inf corners give NaN samples, as in the kernel
        top = g[y0, x0] * (1 - wx) + g[y0, x1] * wx
        bot = g[y1, x0] * (1 - wx) + g[y1, x1] * wx
        return top * (1 - wy) + bot * wy


def _consistent(w, b, alpha, beta):
    s = w + b
    d2 = (s * s).sum(-1)
    rhs = alpha * ((w * w).sum(-1) + (b * b).sum(-1)) + beta
    with np.errstate(invalid="ignore"):
        return (d2 <= rhs) & np.isfinite(rhs)


def aligned(frames, flow_fw, flow_bw, t, radius, t_lo, t_hi, alpha=0.01, beta=0.5):
    """The aligned neighbours of frame t: a list of (H,W,3) float64 arrays, NaN where undefined, forward k = 1..R then
    backward k = 1..R (directions clamped to [t_lo, t_hi])."""
    S, H, W, _ = frames.shape
    al, be = float(np.float32(alpha)), float(np.float32(beta))
    y, x = np.mgrid[0:H, 0:W]
    out = []
    for fwd in (True, False):
        K = min(radius, t_hi - t if fwd else t - t_lo)
        q = np.stack([x.ravel(), y.ravel()], 1).astype(np.float32)
        live = np.ones(H * W, bool)
        for k in range(1, K + 1):
            pair = (t + k - 1 if fwd else t - k) % S
            step, check = (flow_fw[pair], flow_bw[pair]) if fwd else (flow_bw[pair], flow_fw[pair])
            idx = np.nonzero(live)[0]
            w = _sample(step, q[idx, 0].astype(np.float64), q[idx, 1].astype(np.float64))
            with np.errstate(invalid="ignore", over="ignore"):
                nq = q[idx] + w.astype(np.float32)
                ok = (nq[:, 0] >= 0) & (nq[:, 0] <= W - 1) & (nq[:, 1] >= 0) & (nq[:, 1] <= H - 1)
            b = np.full_like(w, np.nan)
            b[ok] = _sample(check, nq[ok, 0].astype(np.float64), nq[ok, 1].astype(np.float64))
            ok &= _consistent(w, b, al, be)
            live[idx[~ok]] = False
            q[idx[ok]] = nq[ok]
            a = np.full((H * W, 3), np.nan)
            keep = idx[ok]
            a[keep] = _sample(frames[(t + k if fwd else t - k) % S], q[keep, 0].astype(np.float64),
                              q[keep, 1].astype(np.float64))
            out.append(a.reshape(H, W, 3))
    return out


def weight(a, ref, sigma, h, patch):
    """(H,W) float64 weight of one aligned neighbour a (NaN = undefined) against the frame ref (H,W,3)."""
    H, W, _ = a.shape
    r = patch
    defined = ~np.isnan(a[..., 0])
    sq = np.where(defined[..., None], (a - ref) ** 2, 0.0).sum(-1)
    pd = np.pad(sq, r)
    pn = np.pad(defined.astype(np.int64), r)
    D, n = np.zeros((H, W)), np.zeros((H, W), np.int64)
    for oy in range(2 * r + 1):
        for ox in range(2 * r + 1):
            D += pd[oy:oy + H, ox:ox + W]
            n += pn[oy:oy + H, ox:ox + W]
    with np.errstate(invalid="ignore", divide="ignore"):
        d2 = D / (3.0 * n)
        hh = h * sigma
        w = np.exp(-np.maximum(d2 - 2.0 * sigma * sigma, 0.0) / (hh * hh)) if np.isfinite(hh) else np.ones_like(d2)
    return np.where(defined, w, 0.0)


def denoise(frames, flow_fw, flow_bw, radius, sigma, h, patch, alpha=0.01, beta=0.5, t0=0, n=None, t_lo=0, t_hi=None,
            flows=None):
    """mfn_denoise_frames in float64.  frames (S,H,W,3) uint8 ring, flow_fw / flow_bw (S,H,W,2) rings; returns
    (n,H,W,3) uint8 for frames t0 .. t0+n-1.  `flows` (a callable t -> list of aligned neighbours) replaces the chain:
    the scene tests give the true alignment through it."""
    frames = np.asarray(frames)
    S = frames.shape[0]
    t_hi = t_lo + S - 1 if t_hi is None else t_hi
    n = t_hi - t0 + 1 if n is None else n
    out = np.empty((n,) + frames.shape[1:], np.uint8)
    sigma = float(np.float32(sigma))
    h = float(np.float32(h)) if np.isfinite(h) else float(h)
    for i in range(n):
        t = t0 + i
        ref = frames[t % S].astype(np.float64)
        nb = flows(t) if flows is not None else aligned(frames, flow_fw, flow_bw, t, radius, t_lo, t_hi, alpha, beta)
        num, den = ref.copy(), np.ones(ref.shape[:2])
        for a in nb:
            w = weight(a, ref, sigma, h, patch)
            num += np.where(w[..., None] > 0, w[..., None] * np.nan_to_num(a), 0.0)
            den += w
        out[i] = np.clip(np.rint(num / den[..., None]), 0, 255).astype(np.uint8)
    return out


def noise_sums(frames):
    f = np.asarray(frames).astype(np.int64)
    if f.ndim == 3:
        f = f[None]
    c = f[:, 1:-1, 1:-1]
    v = (f[:, :-2, :-2] - 2 * f[:, :-2, 1:-1] + f[:, :-2, 2:] - 2 * f[:, 1:-1, :-2] + 4 * c - 2 * f[:, 1:-1, 2:] +
         f[:, 2:, :-2] - 2 * f[:, 2:, 1:-1] + f[:, 2:, 2:])
    return np.abs(v).sum(axis=(1, 2, 3))


def noise_sigma(frames):
    f = np.asarray(frames)
    H, W = f.shape[-3], f.shape[-2]
    S = noise_sums(f)
    s = np.array([SQRT_HALF_PI * float(v) / (18.0 * float(W - 2) * float(H - 2)) for v in S])
    return np.maximum(s, NOISE_FLOOR)
