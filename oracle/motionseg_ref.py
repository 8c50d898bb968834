"""float64 numpy restatement of moving-object segmentation (csrc/motionseg.cu; the rule is in include/maskflow_b200.h,
"Moving-object segmentation"), written from the rule.

    score(res_a, occ_a, res_b, occ_b)    -> s (H,W) float32, NaN where undefined: the smaller defined residual
    label(mask)                          -> (labels (H,W) int64, n): 8-connected components numbered 1..n in raster order
                                            of their first pixel, 0 for the background
    segment(res_a, occ_a, res_b, occ_b, flow_a, affine_a, tau_lo, tau_hi, min_area, max_objects)
                                         -> (labels (N,H,W) uint8, objects (N,max_objects,10) float64, count (N,),
                                            dropped (N,)): the whole rule; either side may be None
    scale_bits(H, W)                     -> S, the kernel's fixed-point scale 2^S of the displacement sums

The labelling works on horizontal runs: the runs of consecutive rows that touch (8-connectivity: overlap or meet at a
corner) are joined by a sparse connected-components pass, and each component is numbered by its first run, which in raster
order holds its first pixel.  It does not use scipy.ndimage; the tests check it against scipy.ndimage.label with a 3x3
structure.  The displacement means are exact sums (math.fsum) over the pixel count.

`control` exists for the tests' controls and changes the rule: "four_connected" (runs must overlap, corners do not join),
"max_score" (s = max(a, b) instead of min(a, b)).
"""
from __future__ import annotations

import math

import numpy as np
from scipy.sparse import coo_matrix
from scipy.sparse.csgraph import connected_components

CONTROLS = ("four_connected", "max_score")
COLUMNS = ("area", "x0", "y0", "x1", "y1", "cx", "cy", "peak", "dx", "dy")
CLAMP = 65536.0


def scale_bits(H, W):
    return 46 - int(H * W).bit_length()


def _defined(res, occ):
    res = np.asarray(res, np.float32)
    return np.where(np.isfinite(res) & (np.asarray(occ) == 0), res, np.float32(np.nan))


def score(res_a, occ_a, res_b, occ_b, control=None):
    a = None if res_a is None else _defined(res_a, occ_a)
    b = None if res_b is None else _defined(res_b, occ_b)
    if a is None and b is None:
        raise ValueError("score: at least one side is needed for the frame's shape")
    if a is None or b is None:
        return a if b is None else b
    return (np.fmax if control == "max_score" else np.fmin)(a, b)      # fmin / fmax: the defined one when one is NaN


def label(mask, control=None):
    m = np.asarray(mask, bool)
    H, W = m.shape
    pad = np.zeros((H, W + 2), np.int8)
    pad[:, 1:-1] = m
    d = np.diff(pad, axis=1)
    row, s = np.nonzero(d == 1)                 # runs in raster order: row, first column ...
    _, e = np.nonzero(d == -1)                  # ... and one past the last column
    e = e - 1
    R = len(row)
    out = np.zeros(H * W, np.int64)
    if R == 0:
        return out.reshape(H, W), 0
    g = 0 if control == "four_connected" else 1
    K = W + 3
    skey, ekey = row * K + s + 1, row * K + e + 1
    lo = np.searchsorted(ekey, (row + 1) * K + (s - g) + 1, "left")       # runs of the next row ending at >= s - g
    hi = np.searchsorted(skey, (row + 1) * K + (e + g) + 1, "right")      # ... and starting at <= e + g
    cnt = np.maximum(hi - lo, 0)
    i = np.repeat(np.arange(R), cnt)
    j = np.repeat(lo, cnt) + (np.arange(len(i)) - np.repeat(np.cumsum(cnt) - cnt, cnt))    # lo[i], lo[i] + 1, ... hi[i] - 1
    graph = coo_matrix((np.ones(len(i), np.int8), (i, j)), shape=(R, R))
    n, comp = connected_components(graph, directed=False)
    _, first = np.unique(comp, return_index=True)          # first run of each component, components in scipy's order
    rank = np.empty(n, np.int64)
    rank[np.argsort(first)] = np.arange(1, n + 1)
    out[np.flatnonzero(m.ravel())] = np.repeat(rank[comp], e - s + 1)
    return out.reshape(H, W), n


def _frame(s, flow, A, a_def, tau_lo, tau_hi, min_area, max_objects, control):
    H, W = s.shape
    with np.errstate(invalid="ignore"):
        fg = s >= np.float32(tau_lo)
    lab, n = label(fg, control)
    rows = np.zeros((max_objects, 10))
    flat = lab.ravel()
    if n == 0:
        return np.zeros((H, W), np.uint8), rows, 0, 0
    area = np.bincount(flat, minlength=n + 1)[1:]
    peak = np.full(n + 1, -np.inf)
    np.maximum.at(peak, flat[flat > 0], s.ravel()[flat > 0].astype(np.float64))
    peak = peak[1:]
    kept = (area >= min_area) & (peak >= float(np.float32(tau_hi)))
    number = np.cumsum(kept)
    K = int(number[-1])
    newlab = np.where(kept & (number <= max_objects), number, 0)
    out = np.concatenate([[0], newlab])[flat].reshape(H, W)
    count = min(K, max_objects)
    y, x = np.mgrid[0:H, 0:W]
    xs, ys, ol = x.ravel(), y.ravel(), out.ravel()
    if flow is not None:
        xf, yf = xs.astype(np.float64), ys.astype(np.float64)
        u, v = flow[..., 0].ravel().astype(np.float64), flow[..., 1].ravel().astype(np.float64)
        ddx = np.clip((xf + u) - ((A[0, 0] * xf + A[0, 1] * yf) + A[0, 2]), -CLAMP, CLAMP)
        ddy = np.clip((yf + v) - ((A[1, 0] * xf + A[1, 1] * yf) + A[1, 2]), -CLAMP, CLAMP)
        adef = a_def.ravel()
    idx = np.flatnonzero(ol)                               # the labelled pixels grouped by label, raster order inside
    idx = idx[np.argsort(ol[idx], kind="stable")]
    bounds = np.searchsorted(ol[idx], np.arange(1, count + 2))
    first = np.flatnonzero(kept)[:count]                   # component of label k + 1
    for k in range(count):
        seg = idx[bounds[k]:bounds[k + 1]]
        c = first[k]
        px, py = xs[seg], ys[seg]
        dx = dy = np.nan
        if flow is not None:
            sa = seg[adef[seg]]
            if len(sa):
                dx = math.fsum(ddx[sa]) / len(sa)
                dy = math.fsum(ddy[sa]) / len(sa)
        rows[k] = (area[c], px.min(), py.min(), px.max(), py.max(), float(px.sum()) / area[c],
                   float(py.sum()) / area[c], peak[c], dx, dy)
    return out.astype(np.uint8), rows, count, K - count


def segment(res_a, occ_a, res_b, occ_b, flow_a=None, affine_a=None, tau_lo=1.0, tau_hi=2.0, min_area=64,
            max_objects=255, control=None):
    ref = res_a if res_a is not None else res_b
    N, H, W = np.asarray(ref).shape
    labels = np.zeros((N, H, W), np.uint8)
    objects = np.zeros((N, max_objects, 10))
    count = np.zeros(N, np.int64)
    dropped = np.zeros(N, np.int64)
    for n in range(N):
        s = score(None if res_a is None else res_a[n], None if occ_a is None else occ_a[n],
                  None if res_b is None else res_b[n], None if occ_b is None else occ_b[n], control)
        a_def = None if res_a is None else np.isfinite(_defined(res_a[n], occ_a[n]))
        labels[n], objects[n], count[n], dropped[n] = _frame(
            s, None if res_a is None else np.asarray(flow_a[n]), None if res_a is None else np.asarray(affine_a[n]),
            a_def, tau_lo, tau_hi, min_area, max_objects, control)
    return labels, objects, count, dropped
