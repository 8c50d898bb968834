"""The comparison of video denoising with oracle/denoise_ref.py (tests/test_denoise.py derives the tolerances), and the
synthetic inputs of its kernel checks."""
import numpy as np
from scipy.ndimage import gaussian_filter

EXACT, FLIPPED = 0.999, 1e-5


def _mismatch(got, ref):
    """(share of values differing by more than 1, share exact, largest difference)."""
    diff = np.abs(np.asarray(got).astype(np.int64) - ref)
    exact = float((diff == 0).mean()) if diff.size else 1.0
    far = float((diff > 1).mean()) if diff.size else 0.0
    return far, exact, int(diff.max(initial=0))


def _check(got, ref, what="", flipped=0.0):
    """|diff| <= 1 with at least EXACT exact, except on at most a share `flipped` of the values (a chain decision taken
    the other way)."""
    far, exact, dmax = _mismatch(got, ref)
    assert far <= flipped and exact >= EXACT, f"{what}: share beyond 1 {far:.2e}, max {dmax}, exact {exact:.6f}"
    return exact


def _case(rng, S, H, W, sigma=8.0):
    """A smooth textured pan with noise, flows of about (0.7, -0.4) px with noise in both directions (most chains run,
    some stop at the round-trip test), NaN and inf spots, and targets that leave the frame.  A 1-pixel-high (or wide)
    frame gets flows along its one row (column)."""
    base = gaussian_filter(rng.integers(0, 256, (H + 8, W + 8, 3)).astype(np.float64), (1.5, 1.5, 0))
    frames = np.clip(np.rint(base[None, 4:4 + H, 4:4 + W] + rng.normal(0, sigma, (S, H, W, 3))), 0, 255).astype(np.uint8)
    fw = rng.normal(0, 0.6, (S, H, W, 2)) + np.array([0.7, -0.4])
    bw = -fw + rng.normal(0, 0.3, (S, H, W, 2))
    bw[rng.random((S, H, W)) < 0.05] += 3.0                      # round trips that fail
    fw[rng.random((S, H, W)) < 0.02] *= 40.0                    # targets far outside
    m = rng.random((S, H, W, 2)) < 0.005
    fw[m] = rng.choice([np.nan, np.inf, -np.inf], int(m.sum()))
    for f in (fw, bw):
        if H == 1:
            f[..., 1] = 0.0
        if W == 1:
            f[..., 0] = 0.0
    return frames, fw.astype(np.float32), bw.astype(np.float32)
