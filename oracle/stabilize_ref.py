"""float64 numpy restatement of video stabilisation (csrc/stabilize.cu and maskflownet_b200/camera.py; the rules are in
include/maskflow_b200.h, "Video stabilisation", and in camera.stabilize_path's docstring), written from the rules.

    fit(flow, iterations, sigma)        -> (affine (N,2,3) float64, ok (N,) bool, residual (N,H,W) float32): the robust
                                           affine camera motion of each flow (IRLS with annealed Cauchy weights)
    warp(src, M)                        -> (N,H,W,3) uint8: src sampled bilinearly at M [x,y,1], clamped to the frame
    path(affine, ok, H, W, radius, crop) -> M (T,2,3): the stabilising warps of a T-frame video from its T-1 pair fits
    corners(A, H, W)                    -> (N,4,2): A applied to the four frame corners, how fits are compared

The kernel sums in a different order (per-thread strided sums, then fixed trees), so its fit differs from this one by
float64 rounding only; the warp's arithmetic is the same expression in the same order, so values differ only where the
kernel's fused multiply-adds move a value across a rounding tie (+-1).

`control` exists for the tests' controls and changes the rule: "swap_xy" (phi = (y^, x^, 1)), "keep_outside" (targets
outside the frame are not excluded), "no_reweight" (the weights stay 1 after iteration 0), "warp_transpose" (the warp
applies M's 2x2 part transposed), "warp_half_pixel" (the warp samples half a pixel off, at M o + (1/2, 1/2)).
"""
from __future__ import annotations

import numpy as np

CONTROLS = ("swap_xy", "keep_outside", "no_reweight", "warp_transpose", "warp_half_pixel")
FIT_CONTROLS = ("swap_xy", "keep_outside", "no_reweight")


def _frame(H, W):
    return 0.5 * (W - 1), 0.5 * (H - 1), 0.5 * max(W, H)


def _solve(m, H, W):
    """(A (2,3), ok) from the 12 sums: M = [[a,b,c],[b,d,e],[c,e,f]], b_x = m[6:9], b_y = m[9:12]."""
    Mm = np.array([[m[0], m[1], m[2]], [m[1], m[3], m[4]], [m[2], m[4], m[5]]])
    det = np.linalg.det(Mm)
    tr3 = np.trace(Mm) / 3.0
    if not (m[5] >= 3.0 and det > 1e-9 * tr3 ** 3):
        return np.array([[1.0, 0.0, 0.0], [0.0, 1.0, 0.0]]), False
    rx, ry = np.linalg.solve(Mm, m[6:9]), np.linalg.solve(Mm, m[9:12])
    cx, cy, s = _frame(H, W)
    L = np.array([[rx[0], rx[1]], [ry[0], ry[1]]])
    t = np.array([cx + s * rx[2], cy + s * ry[2]]) - L @ np.array([cx, cy])
    return np.concatenate([L, t[:, None]], axis=1), True


def fit(flow, iterations=10, sigma=0.5, control=None):
    flow = np.asarray(flow, np.float32)
    N, H, W, _ = flow.shape
    cx, cy, s = _frame(H, W)
    y, x = np.mgrid[0:H, 0:W].astype(np.float64)
    affine = np.zeros((N, 2, 3))
    ok = np.zeros(N, bool)
    residual = np.zeros((N, H, W), np.float32)
    for n in range(N):
        qx, qy = x + flow[n, ..., 0].astype(np.float64), y + flow[n, ..., 1].astype(np.float64)
        with np.errstate(invalid="ignore"):
            if control == "keep_outside":
                valid = np.isfinite(qx) & np.isfinite(qy)
            else:
                valid = (qx >= 0) & (qx <= W - 1) & (qy >= 0) & (qy <= H - 1)
        px, py, ux, uy = ((v[valid] - c) / s for v, c in ((x, cx), (y, cy), (qx, cx), (qy, cy)))
        if control == "swap_xy":
            px, py = py, px
        X, Y, QX, QY = x[valid], y[valid], qx[valid], qy[valid]
        A = np.eye(2, 3)
        for k in range(iterations):
            if k == 0 or control == "no_reweight":
                w = np.ones_like(px)
            else:
                sk = float(np.float32(sigma)) * 2.0 ** max(0, 4 - k)
                r2 = (A[0, 0] * X + A[0, 1] * Y + A[0, 2] - QX) ** 2 + (A[1, 0] * X + A[1, 1] * Y + A[1, 2] - QY) ** 2
                w = 1.0 / (1.0 + r2 / (sk * sk))
            phi = (px, py, np.ones_like(px))
            m = [np.sum(w * phi[i] * phi[j]) for i, j in ((0, 0), (0, 1), (0, 2), (1, 1), (1, 2), (2, 2))]
            m += [np.sum(w * phi[i] * u) for u in (ux, uy) for i in range(3)]
            A, ok[n] = _solve(np.array(m), H, W)
        affine[n] = A
        r = np.full((H, W), np.nan)
        r[valid] = np.hypot(A[0, 0] * X + A[0, 1] * Y + A[0, 2] - QX, A[1, 0] * X + A[1, 1] * Y + A[1, 2] - QY)
        residual[n] = r.astype(np.float32)
    return affine, ok, residual


def corners(A, H, W):
    A = np.asarray(A, np.float64).reshape(-1, 2, 3)
    c = np.array([[0, 0, 1], [W - 1, 0, 1], [0, H - 1, 1], [W - 1, H - 1, 1]], np.float64)
    return np.einsum("nij,kj->nki", A, c)


def warp(src, M, control=None):
    src = np.asarray(src, np.uint8)
    M = np.asarray(M, np.float64).reshape(-1, 2, 3)
    N, H, W, _ = src.shape
    y, x = np.mgrid[0:H, 0:W].astype(np.float64)
    out = np.empty_like(src)
    for n in range(N):
        m = M[n].copy()
        if control == "warp_transpose":
            m[:, :2] = m[:, :2].T
        sx = m[0, 0] * x + m[0, 1] * y + m[0, 2]
        sy = m[1, 0] * x + m[1, 1] * y + m[1, 2]
        if control == "warp_half_pixel":
            sx, sy = sx + 0.5, sy + 0.5
        sx = np.clip(np.nan_to_num(sx, nan=0.0), 0, W - 1)
        sy = np.clip(np.nan_to_num(sy, nan=0.0), 0, H - 1)
        x0, y0 = np.floor(sx).astype(np.int64), np.floor(sy).astype(np.int64)
        x1, y1 = np.minimum(x0 + 1, W - 1), np.minimum(y0 + 1, H - 1)
        wx, wy = (sx - x0)[..., None], (sy - y0)[..., None]
        I = src[n].astype(np.float64)
        top = (1 - wx) * I[y0, x0] + wx * I[y0, x1]
        bot = (1 - wx) * I[y1, x0] + wx * I[y1, x1]
        out[n] = np.clip(np.rint((1 - wy) * top + wy * bot), 0, 255).astype(np.uint8)
    return out


def path(affine, ok, H, W, radius=15, crop=0.9):
    """M_t = P_t S_t^-1 Z: P_0 = I, P_{t+1} = A_t P_t (identity where not ok); S_t the mean of P_s over
    s in [t-R, t+R] & [0, T-1] with weights exp(-d^2 / (2 (R/3)^2)) renormalised (R = 0: S_t = P_t); Z the zoom by crop
    about the frame centre."""
    affine = np.asarray(affine, np.float64).reshape(-1, 2, 3)
    T = len(affine) + 1
    P = [np.eye(3)]
    for a, g in zip(affine, np.asarray(ok, bool)):
        A = np.vstack([a, [0, 0, 1]]) if g else np.eye(3)
        P.append(A @ P[-1])
    cx, cy = 0.5 * (W - 1), 0.5 * (H - 1)
    Z = np.array([[crop, 0, (1 - crop) * cx], [0, crop, (1 - crop) * cy], [0, 0, 1]])
    out = np.empty((T, 2, 3))
    for t in range(T):
        if radius == 0:
            S = P[t]
        else:
            s = np.arange(max(0, t - radius), min(T - 1, t + radius) + 1)
            w = np.exp(-((s - t) ** 2) / (2 * (radius / 3) ** 2))
            S = sum(wi * P[si] for wi, si in zip(w / w.sum(), s))
        out[t] = (P[t] @ np.linalg.inv(S) @ Z)[:2]
    return out
