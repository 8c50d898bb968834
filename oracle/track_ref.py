"""float64 numpy restatement of dense point tracking (csrc/track.cu; the rule is in include/maskflow_b200.h, "Dense point
tracking"), written from the rule.

    texture(frame, h)                     -> lambda2 (Gy,Gx) float64, bit-identical to the kernel's (integers, then one
                                             float64 subtraction and one correctly rounded square root)
    advance(pos, status, flow_fw, flow_bw, alpha, beta, boundary)
                                          -> dict: "status" (K,) uint8 after the advance (EMPTY, TRACKED, LEFT, OCCLUDED,
                                             BOUNDARY), "pos" (K,2) float32 (NaN unless TRACKED), "amb" (K,) bool (a
                                             decision the kernel's fp32 arithmetic may take the other way) and "eq" (K,)
                                             (a bound on |kernel position - "pos"|)
    seed(pos, status, lambda2, lambda_max, queries, frame, h, tau, H, W)
                                          -> (pos, status, dropped) of the frame: query births and the dense seeds, from
                                             the state after the advance
    track(frames, flows_fw, flows_bw, ...) -> (xy (T,K,2) float32, status (T,K) uint8, dropped (T,)): the whole chain

Positions are float32, as the rule defines them: q = float32(p + w), w the bilinear sample at p in float64, so the
oracle's state has the kernel's type.  Everything else (the samples, the round-trip test, the flow gradient) is float64.
The fp32 arithmetic of the kernel may decide a threshold the other way where the float64 value lies within its error
bound; advance() flags those slots ("amb") from bounds built here, next to the arithmetic they bound:
  * a bilinear sample (two fb_lerp levels, each p (1-w) + q w): at most 8 u m off, u = 2^-24, m = the largest |corner|,
    and exact where both weights are 0 (4 u m per level with a non-zero weight);
  * q = fl(p + w): the kernel's and the oracle's differ by at most that plus two ulp of q (none for an exact sample);
  * the backward sample at a q that is off by eq: 8 u mb + 2 mb (|dx| + |dy|), mb the largest |corner| (the
    interpolant's slope is below 2 mb), or of the 4x4 block around floor(q) where q +- eq crosses an integer;
  * |s|^2 and alpha |.|^2 + beta from samples off by e: 2 sqrt(2) |s| e + 2 e^2 per square sum, 4 u relative for the
    float32 sums and products;
  * the gradient sum g of exact flow values: 6 u g.
Seeding reads only the state after the advance, the integer texture and the query rows, so given the kernel's state its
births and dropped count are exact: tests compare them with no exclusion.

`control` exists for the tests' controls and changes the rule: "bw_at_p" (the backward flow sampled at p instead of q),
"no_boundary" (the motion-boundary test dropped), "round_cell" (cell index from rint instead of floor), "ignore_coverage"
(every textured cell is a candidate), "sample_rounded" (flow_fw read at the pixel nearest p instead of sampled).
"""
from __future__ import annotations

import numpy as np

EMPTY, TRACKED, BORN, LEFT, OCCLUDED, BOUNDARY = range(6)
U = 2.0 ** -24
FLT_MAX = float(np.finfo(np.float32).max)
CONTROLS = ("bw_at_p", "no_boundary", "round_cell", "ignore_coverage", "sample_rounded")
ADVANCE_CONTROLS = ("bw_at_p", "no_boundary", "sample_rounded")


def grid(H, W, h):
    return W // h, H // h


def texture(frame, h):
    """lambda2 (Gy,Gx) of one (H,W,3) uint8 frame."""
    I = np.asarray(frame).astype(np.int64).sum(-1)
    H, W = I.shape
    Gx, Gy = grid(H, W, h)
    xs, ys = np.arange(W), np.arange(H)
    gx = I[:, np.minimum(xs + 1, W - 1)] - I[:, np.maximum(xs - 1, 0)]
    gy = I[np.minimum(ys + 1, H - 1), :] - I[np.maximum(ys - 1, 0), :]
    sx, sy = np.arange(Gx) * h + h // 2, np.arange(Gy) * h + h // 2
    a, b, c = (np.zeros((Gy, Gx), np.int64) for _ in range(3))
    for dy in range(-2, 3):
        yy = np.clip(sy + dy, 0, H - 1)
        for dx in range(-2, 3):
            xx = np.clip(sx + dx, 0, W - 1)
            GX, GY = gx[np.ix_(yy, xx)], gy[np.ix_(yy, xx)]
            a, b, c = a + GX * GX, b + GX * GY, c + GY * GY
    a, b, c = a.astype(np.float64), b.astype(np.float64), c.astype(np.float64)
    hh = 0.5 * (a - c)
    l2 = 0.5 * (a + c) - np.sqrt(hh * hh + b * b)
    return np.where(l2 > 0.0, l2, 0.0)


def _sample(plane, qx, qy):
    """(n,2) float64 bilinear samples of the (H,W,2) plane at float64 positions inside the frame, the kernel's corner rule,
    and a bound on the fp32 sample's error over u = 2^-24 (the largest |corner| times 4 per level with a non-zero
    weight)."""
    H, W, _ = plane.shape
    x0, y0 = np.floor(qx).astype(np.int64), np.floor(qy).astype(np.int64)
    x1, y1 = np.minimum(x0 + 1, W - 1), np.minimum(y0 + 1, H - 1)
    wx, wy = (qx - x0)[:, None], (qy - y0)[:, None]
    g = plane.astype(np.float64)
    a, b, c, d = g[y0, x0], g[y0, x1], g[y1, x0], g[y1, x1]
    top, bot = a * (1 - wx) + b * wx, c * (1 - wx) + d * wx
    m = np.max(np.abs(np.stack([a, b, c, d], 1)), axis=(1, 2))
    # a zero weight makes its fb_lerp level exact (p * 1 + q * 0); each other level adds at most 4 u m
    m = m * (4 * (wx[:, 0] != 0) + 4 * (wy[:, 0] != 0))
    return top * (1 - wy) + bot * wy, m


def _block_max(plane, qx, qy):
    """The largest |value| of the 4x4 block floor(q) - 1 .. floor(q) + 2 (clamped) of the plane, per position."""
    H, W, _ = plane.shape
    x0, y0 = np.floor(qx).astype(np.int64), np.floor(qy).astype(np.int64)
    m = np.zeros(len(qx))
    g = np.abs(plane.astype(np.float64)).max(-1)
    for dy in range(-1, 3):
        for dx in range(-1, 3):
            m = np.maximum(m, g[np.clip(y0 + dy, 0, H - 1), np.clip(x0 + dx, 0, W - 1)])
    return m


def _nearest(p, n):
    return np.clip(np.rint(p), 0, n - 1).astype(np.int64)


def advance(pos, status, flow_fw, flow_bw, alpha=0.01, beta=0.5, boundary=(0.01, 0.002), control=None):
    pos, status = np.asarray(pos, np.float32), np.asarray(status, np.uint8)
    H, W, _ = flow_fw.shape
    K = len(status)
    al, be = float(np.float32(alpha)), float(np.float32(beta))
    ab, bb = float(np.float32(boundary[0])), float(np.float32(boundary[1]))
    out = {"status": np.zeros(K, np.uint8), "pos": np.full((K, 2), np.nan, np.float32), "amb": np.zeros(K, bool),
           "eq": np.zeros(K)}
    idx = np.nonzero((status == TRACKED) | (status == BORN))[0]
    if len(idx) == 0:
        return out
    px, py = pos[idx, 0].astype(np.float64), pos[idx, 1].astype(np.float64)
    with np.errstate(all="ignore"):
        if control == "sample_rounded":
            w = flow_fw[_nearest(py, H), _nearest(px, W)].astype(np.float64)
            mw = np.abs(w).max(-1)
        else:
            w, mw = _sample(flow_fw, px, py)
        Ew = U * mw
        q = (np.stack([px, py], 1) + w).astype(np.float32).astype(np.float64)
        qx, qy = q[:, 0], q[:, 1]
        finite = np.isfinite(qx) & np.isfinite(qy)
        # an exact sample gives the kernel's q exactly; otherwise the two float32 roundings add an ulp each
        Eq = np.where(Ew > 0, Ew + 2 * np.spacing(np.abs(q).max(-1).astype(np.float32)).astype(np.float64), 0.0)
        inside = finite & (qx >= 0) & (qx <= W - 1) & (qy >= 0) & (qy <= H - 1)
        surely_in = (qx >= Eq) & (qx <= W - 1 - Eq) & (qy >= Eq) & (qy <= H - 1 - Eq)
        surely_out = (qx < -Eq) | (qx > W - 1 + Eq) | (qy < -Eq) | (qy > H - 1 + Eq)
        amb_left = finite & (Eq > 0) & ~surely_in & ~surely_out          # an exact q is the kernel's
        # the round trip, where the target is inside (clamped elsewhere only to keep the indexing valid)
        cx, cy = np.clip(np.nan_to_num(qx), 0, W - 1), np.clip(np.nan_to_num(qy), 0, H - 1)
        b, eb = _sample(flow_bw, px, py) if control == "bw_at_p" else _sample(flow_bw, cx, cy)
        crosses = (np.floor(cx - Eq) != np.floor(cx + Eq)) | (np.floor(cy - Eq) != np.floor(cy + Eq))
        mb = np.where(crosses, _block_max(flow_bw, cx, cy), eb / 8)   # the kernel's q may pick the neighbouring cell
        Eb = np.where(Eq > 0, 8 * U * mb + 2 * mb * 2 * Eq, U * eb)
        s = w + b
        d2 = (s ** 2).sum(-1)
        wn2, bn2 = (w ** 2).sum(-1), (b ** 2).sum(-1)
        m2 = wn2 + bn2
        rhs = al * m2 + be
        rhs_finite = (m2 <= FLT_MAX) & (rhs <= FLT_MAX)
        consistent = (d2 <= rhs) & rhs_finite
        es = Ew + Eb + U * np.abs(s).max(-1)
        err = (2 * np.sqrt(2) * np.sqrt(d2) * es + 2 * es ** 2 + 3 * U * d2
               + al * (2 * np.sqrt(2) * (np.sqrt(wn2) * Ew + np.sqrt(bn2) * Eb) + 2 * (Ew ** 2 + Eb ** 2) + 4 * U * m2)
               + 2 * U * rhs)
        near_max = ((m2 >= FLT_MAX / 1.01) & (m2 <= FLT_MAX * 1.01)) | ((rhs >= FLT_MAX / 1.01) & (rhs <= FLT_MAX * 1.01))
        amb_occ = ~(np.abs(d2 - rhs) > err) & np.isfinite(d2) & np.isfinite(rhs) | near_max
        # the motion boundary at the pixel nearest p
        nx, ny = _nearest(px, W), _nearest(py, H)
        g = np.zeros(len(idx))
        for (x_a, y_a, x_b, y_b) in ((np.maximum(nx - 1, 0), ny, np.minimum(nx + 1, W - 1), ny),
                                     (nx, np.maximum(ny - 1, 0), nx, np.minimum(ny + 1, H - 1))):
            dist = (x_b - x_a) + (y_b - y_a)
            diff = (flow_fw[y_b, x_b].astype(np.float64) - flow_fw[y_a, x_a]) / np.maximum(dist, 1)[:, None]
            g = g + np.where(dist[:, None] > 0, diff ** 2, 0.0).sum(-1)
        rb = ab * wn2 + bb
        smooth = (g <= rb) | (control == "no_boundary")
        errb = 6 * U * g + ab * (2 * np.sqrt(2) * np.sqrt(wn2) * Ew + 2 * Ew ** 2 + 2 * U * wn2) + 2 * U * rb
        amb_b = ~(np.abs(g - rb) > errb) & np.isfinite(g) & np.isfinite(rb) & (control != "no_boundary")
    st = np.where(~inside, LEFT, np.where(~consistent, OCCLUDED, np.where(~smooth, BOUNDARY, TRACKED))).astype(np.uint8)
    amb = amb_left | ((inside | amb_left) & (amb_occ | ((consistent | amb_occ) & amb_b)))
    out["status"][idx] = st
    tracked = st == TRACKED
    out["pos"][idx[tracked]] = q[tracked].astype(np.float32)
    out["amb"][idx] = amb
    out["eq"][idx] = np.where(np.isfinite(Eq), Eq, np.inf)
    return out


def _cell(p, h, control):
    return (np.rint(p) if control == "round_cell" else np.floor(p)).astype(np.int64) // h


def covered(pos, status, H, W, h, control=None):
    """(Gy,Gx) bool: the cells of the TRACKED and BORN slots."""
    Gx, Gy = grid(H, W, h)
    cov = np.zeros((Gy, Gx), bool)
    live = (status == TRACKED) | (status == BORN)
    i, j = _cell(pos[live, 0].astype(np.float64), h, control), _cell(pos[live, 1].astype(np.float64), h, control)
    ok = (i < Gx) & (j < Gy)
    cov[j[ok], i[ok]] = True
    return cov


def seed(pos, status, lambda2, lambda_max, queries, frame, h, tau, H, W, control=None):
    """The frame's births from the state after its advance (or the reset state, for frame 0)."""
    pos, status = np.array(pos, np.float32), np.array(status, np.uint8)
    queries = np.zeros((0, 3), np.float32) if queries is None else np.asarray(queries, np.float32)
    M = len(queries)
    for i in np.nonzero(queries[:, 0] == np.float32(frame))[0]:
        x, y = queries[i, 1], queries[i, 2]
        if 0 <= x <= W - 1 and 0 <= y <= H - 1:
            pos[i], status[i] = (x, y), BORN
        else:
            pos[i], status[i] = np.nan, LEFT
    cov = covered(pos, status, H, W, h, control)
    if control == "ignore_coverage":
        cov[:] = False
    thr = float(np.float32(tau)) * float(np.asarray(lambda_max).reshape(-1)[0])
    lam = np.asarray(lambda2)
    cand = np.flatnonzero(~cov & (lam > 0) & (lam >= thr))
    free = M + np.flatnonzero(status[M:] == EMPTY)
    n = min(len(cand), len(free))
    Gx = lam.shape[1] if lam.ndim == 2 else 0
    if n:
        j, i = np.divmod(cand[:n], Gx)
        pos[free[:n]] = np.stack([i * h + h // 2, j * h + h // 2], 1)
        status[free[:n]] = BORN
    return pos, status, len(cand) - n


def capacity(H, W, h, max_tracks=None, queries=None):
    Gx, Gy = grid(H, W, h)
    return (0 if queries is None else len(queries)) + (2 * Gx * Gy if max_tracks is None else max_tracks)


def track(frames, flows_fw, flows_bw, spacing=8, tau=0.001, alpha=0.01, beta=0.5, boundary=(0.01, 0.002),
          max_tracks=None, queries=None, control=None):
    """The whole chain over T frames (T,H,W,3) and their T-1 flow pairs (T-1,H,W,2)."""
    T, H, W, _ = frames.shape
    K = capacity(H, W, spacing, max_tracks, queries)
    xy, st, dropped = np.full((T, K, 2), np.nan, np.float32), np.zeros((T, K), np.uint8), np.zeros(T, np.int64)
    pos, status = np.full((K, 2), np.nan, np.float32), np.zeros(K, np.uint8)
    for k in range(T):
        if k:
            a = advance(pos, status, flows_fw[k - 1], flows_bw[k - 1], alpha, beta, boundary,
                        control if control in ADVANCE_CONTROLS else None)
            pos, status = a["pos"], a["status"]
        lam = texture(frames[k], spacing)
        pos, status, dropped[k] = seed(pos, status, lam, lam.max(initial=0.0), queries, k, spacing, tau, H, W, control)
        xy[k], st[k] = pos, status
    return xy, st, dropped
