"""float64 numpy restatement of frame interpolation by occlusion-weighted forward splatting (csrc/interp.cu; the rule is
in include/maskflow_b200.h, mfn_interpolate_frames), written from the rule.

    interpolate(img0, img1, flow_fw, flow_bw, occ_fw, occ_bw, times, occ_weight=0.01)
        -> dict of (N,T,H,W,...) arrays: "frames" uint8 (N,T,H,W,3), "value" float64 (N,T,H,W,3) (the value before rounding:
           colour sum / weight sum, or the blend at a hole), "wsum" (N,T,H,W) (the weight sum), "hole" bool (N,T,H,W),
           "count" (N,T,H,W) (contributions received, zero-weight ones included) and "wnear" (N,T,H,W) (the sum of the
           source weights w, before the bilinear factor b, of the contributions whose target has |qx| < 1 or |qy| < 1:
           the only ones whose fp32 factors 1 - (q - floor q) are not exact).  "count" and "wnear" are what the error
           bound of the kernel's fixed-point and fp32 arithmetic is built from (tests/test_interpolate.py).

The targets are float32, as the rule defines them: float32(float64(x) + float64(t) * float64(u)), which equals the
kernel's fmaf (the product is exact in float64), so every source picks the same corners as in the kernel.  t, 1 - t and
occ_weight are the float32 values the kernel uses; everything after the target is float64, with float64 sums.

`control` exists for the tests' controls and changes the rule: "drop_corner" (no contribution to the corner floor(q) + (1,1)),
"swap_weights" (t and 1 - t swapped in the source weights), "move_by_t" (img1's sources moved by t instead of 1 - t),
"other_mask" (each image weighted by the other image's occlusion mask).
"""
from __future__ import annotations

import numpy as np

HOLE = 2.0 ** -20


def _splat(img, flow, occ, tt, wt, ow, acc, count, wnear, drop_corner=False):
    """Adds one image's sources into acc (N,H,W,4), count and wnear (N,H,W)."""
    N, H, W, _ = img.shape
    y, x = np.mgrid[0:H, 0:W]
    with np.errstate(invalid="ignore", over="ignore"):
        qx = (x + np.float64(tt) * flow[..., 0].astype(np.float64)).astype(np.float32).astype(np.float64)
        qy = (y + np.float64(tt) * flow[..., 1].astype(np.float64)).astype(np.float32).astype(np.float64)
        ok = (qx >= -1) & (qx <= W) & (qy >= -1) & (qy <= H)
    w = np.float64(wt) * np.where(occ != 0, np.float64(ow), 1.0)
    n = np.broadcast_to(np.arange(N)[:, None, None], ok.shape)[ok]
    qx, qy, w, I = qx[ok], qy[ok], w[ok], img[ok].astype(np.float64)
    near = (np.abs(qx) < 1) | (np.abs(qy) < 1)
    x0, y0 = np.floor(qx), np.floor(qy)
    size = N * H * W
    for dy in (0, 1):
        for dx in (0, 1):
            if drop_corner and (dx, dy) == (1, 1):
                continue
            cx, cy = x0 + dx, y0 + dy
            inside = (cx >= 0) & (cx <= W - 1) & (cy >= 0) & (cy <= H - 1)
            b = (1.0 - np.abs(qx - cx)) * (1.0 - np.abs(qy - cy))
            idx = ((n * H + cy.astype(np.int64)) * W + cx.astype(np.int64))[inside]
            bw = (b * w)[inside]
            for c in range(3):
                acc[..., c] += np.bincount(idx, bw * I[inside, c], size).reshape(N, H, W)
            acc[..., 3] += np.bincount(idx, bw, size).reshape(N, H, W)
            count += np.bincount(idx, None, size).reshape(N, H, W).astype(np.int64)
            wnear += np.bincount(idx, (w * near)[inside], size).reshape(N, H, W)


def interpolate(img0, img1, flow_fw, flow_bw, occ_fw, occ_bw, times, occ_weight=0.01, control=None):
    img0, img1 = np.asarray(img0), np.asarray(img1)
    N, H, W, _ = img0.shape
    T = len(times)
    ow = np.float32(occ_weight)
    out = {"frames": np.zeros((N, T, H, W, 3), np.uint8), "value": np.zeros((N, T, H, W, 3)),
           "wsum": np.zeros((N, T, H, W)), "hole": np.zeros((N, T, H, W), bool),
           "count": np.zeros((N, T, H, W), np.int64), "wnear": np.zeros((N, T, H, W))}
    for k, t in enumerate(times):
        t = np.float32(t)
        omt = np.float32(1) - t
        acc = np.zeros((N, H, W, 4))
        count = np.zeros((N, H, W), np.int64)
        wnear = np.zeros((N, H, W))
        w0, w1 = (t, omt) if control == "swap_weights" else (omt, t)
        o0, o1 = (occ_bw, occ_fw) if control == "other_mask" else (occ_fw, occ_bw)
        t1 = t if control == "move_by_t" else omt
        drop = control == "drop_corner"
        _splat(img0, flow_fw, o0, t, w0, ow, acc, count, wnear, drop)
        _splat(img1, flow_bw, o1, t1, w1, ow, acc, count, wnear, drop)
        hole = acc[..., 3] < HOLE
        blend = np.float64(omt) * img0 + np.float64(t) * img1
        with np.errstate(invalid="ignore", divide="ignore"):
            value = np.where(hole[..., None], blend, acc[..., :3] / acc[..., 3:])
        out["frames"][:, k] = np.clip(np.rint(value), 0, 255).astype(np.uint8)
        out["value"][:, k], out["wsum"][:, k], out["hole"][:, k] = value, acc[..., 3], hole
        out["count"][:, k], out["wnear"][:, k] = count, wnear
    return out
