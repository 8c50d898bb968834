"""The camera path of video stabilisation, on the host in float64 numpy.

The GPU fits the camera's motion between consecutive frames (ops.affine_motion) and warps the frames (ops.warp_frames_affine);
in between, this module turns the T-1 pair fits of a T-frame video into one warp per frame.  stabilize_path states the
rule; network.stabilize_video and video.VideoStabilizer both go through it, so the eager and the streamed results are the
same bit for bit.
"""
from __future__ import annotations

import math

import numpy as np

from ._lib import MaskflowError


def check_path_args(radius, crop, who: str) -> None:
    if not (isinstance(radius, (int, np.integer)) and not isinstance(radius, bool) and radius >= 0):
        raise MaskflowError(f"{who}: radius must be a non-negative integer, got {radius!r}")
    try:
        good = 0.0 < float(crop) <= 1.0
    except (TypeError, ValueError):
        good = False
    if not good:
        raise MaskflowError(f"{who}: crop must lie in (0,1], got {crop!r}")


def path_step(P: np.ndarray, affine: np.ndarray, ok) -> np.ndarray:
    """P_{t+1} = A_t o P_t (3x3 homogeneous) from the fit of pair (t, t+1); a failed fit (ok false) counts as the
    identity, so the path holds still over that pair."""
    if not ok:
        return P.copy()
    A = np.eye(3)
    A[:2] = np.asarray(affine, np.float64).reshape(2, 3)
    return A @ P


def zoom(H: int, W: int, crop: float) -> np.ndarray:
    """Z: the zoom by `crop` about the frame centre ((W-1)/2, (H-1)/2), output pixel -> virtual camera pixel."""
    c, cx, cy = float(crop), 0.5 * (W - 1), 0.5 * (H - 1)
    return np.array([[c, 0.0, (1.0 - c) * cx], [0.0, c, (1.0 - c) * cy], [0.0, 0.0, 1.0]])


def stabilize_path(P: np.ndarray, t: int, n: int, H: int, W: int, radius: int = 15, crop: float = 0.9,
                   first: int = 0) -> np.ndarray:
    """The stabilising warp M_t (2,3) float64 of frame t of an n-frame H x W video, which ops.warp_frames_affine applies
    (output pixel -> position in frame t).

    Rule.  A_t is the fit of pair (t, t+1) (ops.affine_motion: frame-t pixel -> its position in frame t+1), the identity
    where the fit failed.  The camera path is P_0 = I, P_{t+1} = A_t P_t (3x3 homogeneous; path_step): P_t maps frame-0
    coordinates to frame t.  The smoothed path is the Gaussian-weighted mean
        S_t = sum_s g_s P_s / sum_s g_s,   s in [t-R, t+R] & [0, n-1],   g_s = exp(-(s-t)^2 / (2 (R/3)^2))
    (renormalised over the truncated window at the ends of the video); R = 0 gives S_t = P_t.  The warp is
        M_t = P_t S_t^-1 Z,
    Z = zoom(H, W, crop), the zoom about the frame centre that keeps the replicated border mostly out of view.  An output
    pixel o thus shows the point of frame t that the smoothed camera sees at Z o.  With R = 0, M_t = Z exactly.

    P holds P_first .. P_{first+len(P)-1} (at least the window of t); the sum runs over the window in increasing s, so a
    caller holding only the window gets the same bits as one holding the whole path."""
    check_path_args(radius, crop, "stabilize_path")
    Z = zoom(H, W, crop)
    if radius == 0:
        return Z[:2].copy()
    lo, hi = max(0, t - radius), min(n - 1, t + radius)
    if lo < first or hi >= first + len(P):
        raise MaskflowError(f"stabilize_path: frame {t} needs P_{lo}..P_{hi}, given P_{first}..P_{first + len(P) - 1}")
    two_var = 2.0 * (radius / 3.0) ** 2
    g = [math.exp(-float((s - t) ** 2) / two_var) for s in range(lo, hi + 1)]
    tot = sum(g)
    S = np.zeros((3, 3))
    for gi, s in zip(g, range(lo, hi + 1)):
        S += (gi / tot) * P[s - first]
    return (P[t - first] @ np.linalg.inv(S) @ Z)[:2]


def camera_path(affine, ok, H: int, W: int, radius: int = 15, crop: float = 0.9) -> np.ndarray:
    """M (T,2,3) float64 for a T-frame video from its T-1 pair fits, affine (T-1,2,3) and ok (T-1,) (stabilize_path)."""
    check_path_args(radius, crop, "camera_path")
    affine = np.asarray(affine, np.float64).reshape(-1, 2, 3)
    ok = np.asarray(ok).reshape(-1)
    if len(ok) != len(affine):
        raise MaskflowError(f"camera_path: {len(affine)} fits but {len(ok)} ok flags")
    P = [np.eye(3)]
    for a, g in zip(affine, ok):
        P.append(path_step(P[-1], a, bool(g)))
    n = len(P)
    return np.stack([stabilize_path(P, t, n, H, W, radius, crop) for t in range(n)])
