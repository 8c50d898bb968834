"""The comparison of frame interpolation results with oracle/interp_ref.py, with the rounding-tie exclusions."""
import numpy as np

from oracle import interp_ref

from .bounds import U


EXCLUDED_MAX = 1e-3           # share of the compared values that may be excluded as near a rounding tie
DB = 2.0 ** -23


def _ambiguous(ref, H, W, img0, img1, times):
    """(N,T,H,W,3) bool: values whose rounding the kernel's arithmetic may decide the other way (module docstring), and
    the part of them where the hole decision itself may go the other way."""
    s_w = 61 - int(2 * H * W).bit_length()
    s_c = s_w - 8
    Wo, n, wnear = ref["wsum"], ref["count"], ref["wnear"]
    dW = DB * wnear + 3 * U * Wo + n * 2.0 ** -(s_w + 1)
    with np.errstate(divide="ignore", invalid="ignore"):
        E = (255 * (DB * wnear + 4 * U * Wo) + n * 2.0 ** -s_c) / (Wo - dW) + 2.0 ** -16
    E = np.where(Wo - dW > 0, E, np.inf)[..., None]
    t = np.asarray(times, np.float32)[None, :, None, None, None]
    i0, i1 = img0[:, None].astype(np.float32), img1[:, None].astype(np.float32)
    blend32 = (t.astype(np.float64) * i1 + (np.float32(1) - t) * i0).astype(np.float32)   # the kernel's fmaf, exactly
    v = ref["value"]
    hole = ref["hole"][..., None]
    near_tie = np.where(hole, np.rint(blend32) != np.rint(v), np.abs(v - (np.floor(v) + 0.5)) <= E)
    near_hole = (np.abs(Wo - interp_ref.HOLE) <= dW)[..., None]
    return near_tie | near_hole, np.broadcast_to(near_hole, near_tie.shape)


def _mismatch(got, ref, img0, img1, times):
    """(values that differ outside the ambiguous ones, values excluded, values compared, max |got - ref| outside the
    values whose hole decision is ambiguous: there one side is the blend and the other the splatted colour)."""
    want = ref["frames"]
    assert got.shape == want.shape and got.dtype == np.uint8, (got.shape, want.shape, got.dtype)
    amb, near_hole = _ambiguous(ref, img0.shape[1], img0.shape[2], img0, img1, times)
    diff = np.abs(got.astype(np.int64) - want)
    return int(((diff != 0) & ~amb).sum()), int(amb.sum()), amb.size, int(diff[~near_hole].max(initial=0))


def _check(got, ref, img0, img1, times, what=""):
    bad, excl, total, dmax = _mismatch(got, ref, img0, img1, times)
    assert bad == 0, f"{what}: {bad} values differ from the oracle outside the {excl} ambiguous ones"
    assert dmax <= 1, f"{what}: max |got - ref| = {dmax}"
    return excl, total
