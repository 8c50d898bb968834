"""The comparison of the tracker's advance and seed steps with oracle/track_ref.py."""
import numpy as np

from oracle import track_ref as R


EXCLUDED_MAX = 1e-3
CONSTS = dict(alpha=0.01, beta=0.5, boundary=(0.01, 0.002))


class Tally:
    def __init__(self):
        self.excluded = self.compared = 0

    def check(self):
        print(f"excluded {self.excluded} of {self.compared} slot decisions")
        assert self.excluded <= EXCLUDED_MAX * max(self.compared, 1), (self.excluded, self.compared)


def _compare_advance(prev_pos, prev_status, adv_pos, adv_status, ffw, fbw, tally, control=None, what=""):
    """Mismatching slots outside the exclusions (0 for the kernel against its own rule)."""
    ref = R.advance(prev_pos, prev_status, ffw, fbw, **CONSTS, control=control)
    live = (prev_status == R.TRACKED) | (prev_status == R.BORN)
    amb = ref["amb"]
    bad = (adv_status != ref["status"]) & ~amb
    both = (adv_status == R.TRACKED) & (ref["status"] == R.TRACKED)
    dev = np.abs(adv_pos.astype(np.float64) - ref["pos"]).max(-1)
    bad |= both & ~(dev <= ref["eq"])
    bad |= ~both & (adv_status != R.TRACKED) & ~np.all(np.isnan(adv_pos), -1)
    if tally is not None:
        tally.excluded += int((amb & live).sum())
        tally.compared += int(live.sum())
    return int(bad.sum())


def _compare_seed(adv_pos, adv_status, lam, lmax, q, k, h, tau, H, W, xy, st, dropped, control=None):
    """Mismatching slots and dropped counts of the seeding of frame k against the oracle from the state after the advance
    (exact: no exclusion)."""
    rp, rs, rd = R.seed(adv_pos, adv_status, lam, lmax, q, k, h, tau, H, W, control)
    same = (rs == st) & ((rp == xy) | (np.isnan(rp) & np.isnan(xy))).all(-1)
    return int((~same).sum()) + int(rd != dropped)
