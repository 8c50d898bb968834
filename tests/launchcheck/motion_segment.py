"""The comparison of motion-segmentation results with oracle/motionseg_ref.py."""
import numpy as np

from oracle import motionseg_ref as R


def _mismatch(got, ref, H, W):
    """A description of the first difference between two results (labels, objects, count, dropped), or None."""
    (gl, go, gc, gd), (rl, ro, rc, rd) = got, ref
    gl, go, gc, gd = (np.asarray(v) for v in (gl, go, gc, gd))
    if not np.array_equal(gc, rc) or not np.array_equal(gd, rd):
        return f"count {gc} != {rc} or dropped {gd} != {rd}"
    bad = np.flatnonzero((gl != rl).reshape(len(gl), -1).any(1))
    if len(bad):
        return f"labels differ in frames {bad.tolist()}: {int((gl != rl).sum())} pixels"
    if not np.array_equal(go[..., :8], ro[..., :8]):
        return f"area/box/centroid/peak differ by {np.abs(go[..., :8] - ro[..., :8]).max()}"
    gn, rn = np.isnan(go[..., 8:]), np.isnan(ro[..., 8:])
    if not np.array_equal(gn, rn):
        return "dx/dy NaN pattern differs"
    tol = 2.0 ** -(R.scale_bits(H, W) + 1) + 2.0 ** -50 * (1 + np.abs(np.nan_to_num(ro[..., 8:])))
    err = np.abs(np.nan_to_num(go[..., 8:]) - np.nan_to_num(ro[..., 8:]))
    if (err > tol).any():
        return f"dx/dy differ by {err.max()} > {tol.max()}"
    return None


def _check(got, ref, H, W, what=""):
    m = _mismatch(got, ref, H, W)
    assert m is None, f"{what}: {m}"
