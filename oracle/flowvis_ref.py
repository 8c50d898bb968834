"""float64 restatement of the Middlebury flow colour coding (Baker et al.; the flow_vis.flow_to_color convention that the
reference's predict_new_data.py writes).  TEST INFRASTRUCTURE ONLY: the product computes it in csrc/flowvis.cu.

  make_colorwheel   the 55-entry wheel: segments RY 15, YG 6, GC 4, CB 11, BM 13, MR 6
  flow_to_color     (N,H,W,2) or (H,W,2) (x,y) flow -> (uint8 colours of the same leading shape + 3, rad_max (N,) or scalar)
"""
from __future__ import annotations

import numpy as np


def make_colorwheel() -> np.ndarray:
    RY, YG, GC, CB, BM, MR = 15, 6, 4, 11, 13, 6
    wheel = np.zeros((RY + YG + GC + CB + BM + MR, 3))
    col = 0
    for length, ch, rising, fixed in ((RY, 1, True, (0,)), (YG, 0, False, (1,)), (GC, 2, True, (1,)),
                                      (CB, 1, False, (2,)), (BM, 0, True, (2,)), (MR, 2, False, (0,))):
        ramp = np.floor(255 * np.arange(length) / length)
        wheel[col:col + length, ch] = ramp if rising else 255 - ramp
        for c in fixed:
            wheel[col:col + length, c] = 255
        col += length
    return wheel


def flow_uv_to_colors(u: np.ndarray, v: np.ndarray, bgr: bool = False) -> np.ndarray:
    """Colours of an already normalised flow (u, v) of any shape."""
    wheel = make_colorwheel()
    ncols = wheel.shape[0]
    rad = np.sqrt(u * u + v * v)
    a = np.arctan2(-v, -u) / np.pi
    fk = (a + 1) / 2 * (ncols - 1)
    k0 = np.floor(fk).astype(np.int64)
    k1 = k0 + 1
    k1[k1 == ncols] = 0
    f = fk - k0
    out = np.zeros(u.shape + (3,), np.uint8)
    for i in range(3):
        col = ((1 - f) * wheel[k0, i] + f * wheel[k1, i]) / 255.0
        inside = rad <= 1
        col = np.where(inside, 1 - rad * (1 - col), col * 0.75)
        out[..., 2 - i if bgr else i] = np.floor(255 * col)
    return out


def flow_to_color(flow, max_radius=None, bgr=False):
    """max_radius None (or <= 0): each sample is divided by (its largest radius + 1e-5), the reference's behaviour; else by
    max_radius.  Returns (rgb uint8, rad_max: the radius each sample was normalised by)."""
    flow = np.asarray(flow, np.float64)
    single = flow.ndim == 3
    if single:
        flow = flow[None]
    u, v = flow[..., 0], flow[..., 1]
    if max_radius is None or max_radius <= 0:
        rad_max = np.sqrt(u * u + v * v).max(axis=(1, 2))
        d = rad_max + 1e-5
    else:
        rad_max = np.full(flow.shape[0], float(max_radius))
        d = rad_max
    rgb = flow_uv_to_colors(u / d[:, None, None], v / d[:, None, None], bgr)
    return (rgb[0], rad_max[0]) if single else (rgb, rad_max)
