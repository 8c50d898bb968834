"""The float64 restatement of the forward-backward occlusion test (ops.flow_consistency)."""
import numpy as np


ALPHA, BETA = 0.01, 0.5
AMBIGUOUS_MAX = 1e-3          # share of the compared pixels that may be excluded as ambiguous


def _lerp(p, q, w):
    return p * (1.0 - w) + q * w


def _one_direction(flow, other, alpha, beta):
    """occ (N,H,W) bool and ambiguous (N,H,W) bool for the pixels of `flow` against `other`.  The target x + u is the
    float32 sum, as the rule defines it (one exactly specified rounding: where the other flow is steep, the bilinear
    sample moves with the target's last bit); everything after it is float64."""
    N, H, W, _ = flow.shape
    y, x = np.mgrid[0:H, 0:W]
    with np.errstate(invalid="ignore", over="ignore"):
        qx = (x.astype(np.float32) + flow[..., 0]).astype(np.float64)
        qy = (y.astype(np.float32) + flow[..., 1]).astype(np.float64)
    f = flow.astype(np.float64)
    g = other.astype(np.float64)
    with np.errstate(invalid="ignore", over="ignore"):
        inside = (qx >= 0) & (qx <= W - 1) & (qy >= 0) & (qy <= H - 1)
        sx, sy = np.where(inside, qx, 0.0), np.where(inside, qy, 0.0)
        x0, y0 = np.floor(sx).astype(np.int64), np.floor(sy).astype(np.int64)
        x1, y1 = np.minimum(x0 + 1, W - 1), np.minimum(y0 + 1, H - 1)
        wx, wy = sx - x0, sy - y0
        n = np.arange(N)[:, None, None]
        a, b, c, d = g[n, y0, x0], g[n, y0, x1], g[n, y1, x0], g[n, y1, x1]
        bu = _lerp(_lerp(a[..., 0], b[..., 0], wx), _lerp(c[..., 0], d[..., 0], wx), wy)
        bv = _lerp(_lerp(a[..., 1], b[..., 1], wx), _lerp(c[..., 1], d[..., 1], wx), wy)
        u, v = f[..., 0], f[..., 1]
        d2 = (u + bu) ** 2 + (v + bv) ** 2
        rhs = alpha * (u * u + v * v + bu * bu + bv * bv) + beta
        occ = ~inside | ~(d2 <= rhs) | ~np.isfinite(rhs)
        near_rule = inside & (np.abs(d2 - rhs) <= 1e-4 * (d2 + rhs))
        near_bound = np.minimum.reduce([np.abs(qx), np.abs(qx - (W - 1)), np.abs(qy), np.abs(qy - (H - 1))]) <= 1e-3
    return occ, near_rule | near_bound


def consistency_ref(flow_fw, flow_bw, alpha=ALPHA, beta=BETA):
    """(occ_fw, occ_bw, ambiguous_fw, ambiguous_bw) of (N,H,W,2) float32 flows."""
    occ_fw, amb_fw = _one_direction(flow_fw, flow_bw, alpha, beta)
    occ_bw, amb_bw = _one_direction(flow_bw, flow_fw, alpha, beta)
    return occ_fw, occ_bw, amb_fw, amb_bw
