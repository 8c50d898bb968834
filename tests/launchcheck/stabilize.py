"""The comparison of the camera-motion fit and the frame warp with oracle/stabilize_ref.py."""
import numpy as np

from oracle import stabilize_ref as R


CORNER_TOL, RES_TOL, WARP_EXACT = 1e-6, 1e-5, 0.999


def _fit_mismatch(got, ref, H, W):
    """(max corner distance in px, ok flags differ, residual values outside tolerance or NaN pattern differs)."""
    (ga, gok, gres), (ra, rok, rres) = got, ref
    d = float(np.abs(R.corners(ga, H, W) - R.corners(ra, H, W)).max(initial=0.0))
    okbad = not np.array_equal(np.asarray(gok, bool), np.asarray(rok, bool))
    resbad = 0
    if gres is not None:
        gn, rn = np.isnan(gres), np.isnan(rres)
        tol = RES_TOL + np.spacing(np.abs(np.nan_to_num(rres)).astype(np.float32))
        resbad = int((gn != rn).sum() + ((np.abs(np.nan_to_num(gres) - np.nan_to_num(rres)) > tol) & ~gn & ~rn).sum())
    return d, okbad, resbad


def _check_fit(got, ref, H, W, what=""):
    d, okbad, resbad = _fit_mismatch(got, ref, H, W)
    assert not okbad, f"{what}: ok {got[1]} != {ref[1]}"
    assert d <= CORNER_TOL, f"{what}: corners differ by {d} px"
    assert resbad == 0, f"{what}: {resbad} residual values differ"
    return d


def _warp_mismatch(got, ref):
    diff = np.abs(got.astype(np.int64) - ref)
    return int(diff.max(initial=0)), float((diff == 0).mean()) if diff.size else 1.0


def _check_warp(got, ref, what=""):
    dmax, exact = _warp_mismatch(got, ref)
    assert dmax <= 1 and exact >= WARP_EXACT, f"{what}: max |diff| {dmax}, exact {exact:.5f}"
    return exact
