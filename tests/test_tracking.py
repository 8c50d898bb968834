"""Dense point tracking: the kernels (csrc/track.cu, ops.track_*), network.track_video, video.VideoTracker,
video.collect_tracks and tools/track_video.py.

CPU: the kernel source compiled for the host (tests/host_emu/track_emu.cpp) against the float64 oracle
(oracle/track_ref.py): the texture bit for bit, the advance per step from the kernel's previous state, the seeding with no
exclusion; known answers, the synthetic occlusion scene through the oracle and the host kernels, five controls that must
fail the comparison, argument errors and the host bookkeeping.  GPU: the same through the ops at the video sizes, the
video tracker bit for bit against network.track_video, the scene from the kernels, and the command line.

Exclusions (oracle/track_ref.py derives the bounds next to the arithmetic): where the float64 value of a threshold test
(frame bound, round trip, motion boundary) lies within the kernel's fp32 error bound of the threshold, that slot's status
is excluded and counted; at most EXCLUDED_MAX of the compared slots may be.  Every other status must match, and every
TRACKED position must lie within its bound of the oracle's.  The seeding starts from the kernel's own state after the
advance, so its births and dropped counts are compared exactly.
"""
import ctypes
import importlib.util
import os

import numpy as np
import pytest
import torch

from maskflownet_b200 import MaskflowError, _lib, network, ops
from maskflownet_b200.video import TrackFrame, VideoTracker, collect_tracks, track_frames
from oracle import track_ref as R

from launchcheck.emu import build, ptr
from launchcheck.inputs import _deterministic
from launchcheck.tracking import CONSTS, Tally, _compare_advance, _compare_seed

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


# ---------------------------------------------------------------------------------------------------------------
# the host build
# ---------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    L = build(tmp_path_factory, "track_emu")
    v, i, f = ctypes.c_void_p, ctypes.c_int, ctypes.c_float
    L.emu_track_texture.argtypes = [v, v, v, i, i, i, i]
    L.emu_track_advance.argtypes = [v] * 5 + [i] * 4 + [f] * 4
    L.emu_track_seed.argtypes = [v, v, v, i, v, v, v, v, v, i, i, i, i, f]
    return L


class HostTracker:
    """The kernels' launch sequence on the host, with the state in numpy arrays."""

    def __init__(self, L, H, W, spacing=8, tau=0.001, max_tracks=None, queries=None, alpha=0.01, beta=0.5,
                 boundary=(0.01, 0.002)):
        self.L, self.H, self.W, self.h, self.tau = L, H, W, spacing, tau
        self.alpha, self.beta, self.boundary = alpha, beta, boundary
        self.q = np.zeros((0, 3), np.float32) if queries is None else np.ascontiguousarray(queries, np.float32)
        self.M = len(self.q)
        self.K = R.capacity(H, W, spacing, max_tracks, queries)
        self.Gx, self.Gy = R.grid(H, W, spacing)
        self.pos = np.full((self.K, 2), np.nan, np.float32)
        self.status = np.zeros(self.K, np.uint8)
        self.cells = np.zeros(max(self.Gx * self.Gy, 1), np.uint8)
        self.frame = np.zeros(1, np.int32)
        self.dropped = np.zeros(1, np.int32)

    def texture(self, frame):
        lam = np.zeros((1, self.Gy, self.Gx))
        lmax = np.zeros(1)
        self.L.emu_track_texture(ptr(np.ascontiguousarray(frame[None])), ptr(lam), ptr(lmax), 1, self.H, self.W, self.h)
        return lam[0], lmax

    def advance(self, ffw, fbw):
        ab, bb = self.boundary
        self.L.emu_track_advance(ptr(np.ascontiguousarray(ffw)), ptr(np.ascontiguousarray(fbw)), ptr(self.pos),
                                 ptr(self.status), ptr(self.cells), self.K, self.H, self.W, self.h, self.alpha,
                                 self.beta, ab, bb)

    def seed(self, lam, lmax):
        self.L.emu_track_seed(ptr(np.ascontiguousarray(lam)), ptr(lmax), ptr(self.q) if self.M else None, self.M,
                              ptr(self.pos), ptr(self.status), ptr(self.cells), ptr(self.frame), ptr(self.dropped),
                              self.K, self.H, self.W, self.h, self.tau)
        return self.pos.copy(), self.status.copy(), int(self.dropped[0])


class GpuTracker:
    """The same through the ops on the device."""

    def __init__(self, H, W, spacing=8, tau=0.001, max_tracks=None, queries=None, alpha=0.01, beta=0.5,
                 boundary=(0.01, 0.002)):
        self.st = ops.TrackState(H, W, spacing, tau, alpha, beta, boundary, max_tracks, queries)
        self.H, self.W, self.h, self.tau, self.M, self.K = H, W, spacing, tau, self.st.M, self.st.K
        self.q = self.st.queries.cpu().numpy()

    @property
    def pos(self):
        return self.st.pos.cpu().numpy()

    @property
    def status(self):
        return self.st.status.cpu().numpy()

    def texture(self, frame):
        lam, lmax = ops.track_texture(torch.from_numpy(np.ascontiguousarray(frame)).cuda(), self.h)
        return lam, lmax

    def advance(self, ffw, fbw):
        ops.track_advance(self.st, torch.from_numpy(np.ascontiguousarray(ffw)).cuda(),
                          torch.from_numpy(np.ascontiguousarray(fbw)).cuda())

    def seed(self, lam, lmax):
        xy, status, dropped = ops.track_seed(self.st, lam, lmax)
        return xy.cpu().numpy(), status.cpu().numpy(), int(dropped.item())


def _texture_np(tr, frame):
    lam, lmax = tr.texture(frame)
    if isinstance(lam, torch.Tensor):
        return lam, lmax, lam.cpu().numpy(), lmax.cpu().numpy()
    return lam, lmax, lam, lmax


# ---------------------------------------------------------------------------------------------------------------
# the comparison against the oracle, one frame at a time from the kernel's own previous state
# ---------------------------------------------------------------------------------------------------------------
def _run_chain(tr, frames, ffw, fbw, tally=None, control=None):
    """Runs a tracker over the frames; checks every advance (with exclusions) and every seeding (exact) against the
    oracle from the tracker's previous state.  Returns (xy (T,K,2), status (T,K), dropped (T,), mismatches)."""
    T = len(frames)
    xy, st, dropped = np.zeros((T, tr.K, 2), np.float32), np.zeros((T, tr.K), np.uint8), np.zeros(T, np.int64)
    bad = 0
    for k in range(T):
        if k:
            prev_pos, prev_status = xy[k - 1], st[k - 1]
            tr.advance(ffw[k - 1], fbw[k - 1])
            adv_pos, adv_status = tr.pos.copy(), tr.status.copy()
            bad += _compare_advance(prev_pos, prev_status, adv_pos, adv_status, ffw[k - 1], fbw[k - 1], tally,
                                    control if control in R.ADVANCE_CONTROLS else None)
        else:
            adv_pos, adv_status = np.full((tr.K, 2), np.nan, np.float32), np.zeros(tr.K, np.uint8)
        lam, lmax, lam_np, lmax_np = _texture_np(tr, frames[k])
        assert np.array_equal(lam_np, R.texture(frames[k], tr.h)), k
        assert lmax_np[0] == R.texture(frames[k], tr.h).max(initial=0.0), k
        xy[k], st[k], dropped[k] = tr.seed(lam, lmax)
        bad += _compare_seed(adv_pos, adv_status, lam_np, lmax_np, tr.q, k, tr.h, tr.tau, tr.H, tr.W, xy[k], st[k],
                             dropped[k], control if control not in R.ADVANCE_CONTROLS else None)
    return xy, st, dropped, bad


# ---------------------------------------------------------------------------------------------------------------
# inputs
# ---------------------------------------------------------------------------------------------------------------
def _textured(rng, T, H, W, flat=True):
    from scipy.ndimage import gaussian_filter
    f = np.stack([gaussian_filter(rng.standard_normal((H, W, 3)), (1.0, 1.0, 0)) for _ in range(T)])
    f = np.rint((f - f.min()) / max(f.max() - f.min(), 1e-9) * 255).astype(np.uint8)
    if flat:
        f[:, : H // 4, : W // 4] = 128                    # a flat corner: no texture there
    return f


def _flows(rng, T, H, W, special=True):
    """T-1 flow pairs: smooth motion of a few pixels with noise; with `special`, targets on the last row and column,
    exact integers, huge and non-finite values."""
    from scipy.ndimage import gaussian_filter
    out = []
    y, x = np.mgrid[0:H, 0:W]
    for _ in range(2):
        f = np.stack([gaussian_filter(rng.standard_normal((T - 1, H, W)), (0, 4, 4)) * 30 + rng.normal(0, 1.5)
                      for _ in range(2)], -1) + rng.normal(0, 0.05, (T - 1, H, W, 2))
        if special:
            m = rng.random((T - 1, H, W)) < 0.03
            f[..., 0] = np.where(m, (W - 1) - x, f[..., 0])                        # x + u = W - 1 from a pixel
            m = rng.random((T - 1, H, W)) < 0.03
            f[..., 1] = np.where(m, (H - 1) - y, f[..., 1])
            m = rng.random((T - 1, H, W, 2)) < 0.05
            f[m] = rng.integers(-3, 4, int(m.sum()))
            m = rng.random((T - 1, H, W, 2)) < 0.003
            f[m] = rng.choice([np.nan, np.inf, -np.inf, 1e30, -1e30], int(m.sum()))
        out.append(f.astype(np.float32))
    return out


SHAPES = [(1, 1), (1, 29), (23, 1), (37, 53)]


# ---------------------------------------------------------------------------------------------------------------
# CPU: the kernel source on the host
# ---------------------------------------------------------------------------------------------------------------
def test_texture_bit_identical_on_host(emu):
    rng = np.random.default_rng(0)
    for H, W in SHAPES + [(40, 64)]:
        for h in (1, 3, 8):
            for frame in (rng.integers(0, 256, (H, W, 3), dtype=np.uint8), _textured(rng, 1, H, W)[0],
                          np.full((H, W, 3), 255, np.uint8)):
                tr = HostTracker(emu, H, W, h)
                lam, lmax = tr.texture(frame)
                ref = R.texture(frame, h)
                assert np.array_equal(lam, ref) and lmax[0] == ref.max(initial=0.0), (H, W, h)


@pytest.mark.parametrize("H,W", SHAPES, ids=[f"{h}x{w}" for h, w in SHAPES])
def test_chain_matches_oracle_on_host(emu, H, W):
    rng = np.random.default_rng(H * 100 + W)
    T = 6
    frames = _textured(rng, T, H, W)
    ffw, fbw = _flows(rng, T, H, W)
    tally = Tally()
    for h in (1, 4, 8):
        q = np.array([[0, 0, 0], [1, W - 1, H - 1], [2, W / 2, H / 2], [3, W, 0]], np.float32)
        for kw in (dict(), dict(queries=q), dict(max_tracks=3, queries=q)):
            tr = HostTracker(emu, H, W, h, **kw)
            *_, bad = _run_chain(tr, frames, ffw, fbw, tally)
            assert bad == 0, (h, kw)
    tally.check()


def test_advance_with_special_positions_on_host(emu):
    """Live slots at exact integers, on the last row and column and in the partial cells, against flows with NaN, +-inf,
    1e30 and targets on the last row and column."""
    rng = np.random.default_rng(2)
    H, W, K = 37, 53, 4000
    ffw, fbw = (f[0] for f in _flows(rng, 2, H, W))
    pos = np.stack([rng.uniform(0, W - 1, K), rng.uniform(0, H - 1, K)], 1).astype(np.float32)
    pos[:500] = np.rint(pos[:500])
    pos[500:700, 0] = W - 1
    pos[700:900, 1] = H - 1
    pos[900:1000] = (W - 1, H - 1)
    status = rng.choice([R.EMPTY, R.TRACKED, R.BORN, R.LEFT, R.OCCLUDED, R.BOUNDARY], K,
                        p=[0.05, 0.5, 0.3, 0.05, 0.05, 0.05]).astype(np.uint8)
    tally = Tally()
    for h in (1, 8):
        tr = HostTracker(emu, H, W, h, max_tracks=K)
        tr.pos[:], tr.status[:] = pos, status
        tr.advance(ffw, fbw)
        assert _compare_advance(pos, status, tr.pos, tr.status, ffw, fbw, tally) == 0, h
        cells = np.zeros((tr.Gy, tr.Gx), bool)                       # the occupancy map the advance wrote
        t = tr.status == R.TRACKED
        i, j = np.floor(tr.pos[t, 0]).astype(int) // h, np.floor(tr.pos[t, 1]).astype(int) // h
        ok = (i < tr.Gx) & (j < tr.Gy)
        cells[j[ok], i[ok]] = True
        assert np.array_equal(tr.cells[:tr.Gx * tr.Gy].reshape(tr.Gy, tr.Gx).astype(bool), cells), h
        assert set(np.unique(tr.status[t == 0])) <= {R.EMPTY, R.LEFT, R.OCCLUDED, R.BOUNDARY}
    tally.check()


# ---------------------------------------------------------------------------------------------------------------
# known answers (any tracker with texture / advance / seed; no exclusion)
# ---------------------------------------------------------------------------------------------------------------
def _known_answers(make):
    rng = np.random.default_rng(7)
    H, W, h, T = 48, 64, 8, 6
    frames = _textured(rng, 1, H, W).repeat(T, 0)
    frames[:, : H // 4, : W // 4] = 128
    z = np.zeros((T - 1, H, W, 2), np.float32)

    # zero flow: nothing stops, and after frame 0 every textured cell stays covered
    xy, st, dr, bad = _run_chain(make(H, W, h), frames, z, z)
    assert bad == 0
    born0 = st[0] == R.BORN
    assert born0.sum() > 0 and np.all(st[1:][:, born0] == R.TRACKED) and np.all(st[1:][:, ~born0] == R.EMPTY)
    assert np.array_equal(xy[-1][born0], xy[0][born0]) and np.all(dr == 0)

    # an integer translation by (3, 2) per frame: exact positions; tracks that leave the frame end LEFT; the uncovered
    # strip is reseeded
    d = np.array([3, 2], np.float32)
    fw = np.broadcast_to(d, z.shape).copy()
    xy, st, dr, bad = _run_chain(make(H, W, h), _textured(rng, 1, H, W, flat=False).repeat(T, 0), fw, -fw)
    assert bad == 0
    for k in range(1, T):
        alive_before = (st[k - 1] == R.TRACKED) | (st[k - 1] == R.BORN)
        tgt = xy[k - 1][alive_before] + d
        inside = (tgt[:, 0] <= W - 1) & (tgt[:, 1] <= H - 1)
        assert np.all(st[k][alive_before][inside] == R.TRACKED)
        assert np.array_equal(xy[k][alive_before][inside], tgt[inside])
        assert np.all(st[k][alive_before][~inside] == R.LEFT)
        assert np.all(np.isnan(xy[k][alive_before][~inside]))
        born = xy[k][st[k] == R.BORN]
        assert np.all((born[:, 0] < 3 * k + h) | (born[:, 1] < 2 * k + h)), k    # the uncovered strips only
    assert np.any(st[2:] == R.BORN)                                  # the first cells are uncovered from frame 2 on

    # a flat frame: no seeds at all
    flat = np.full((T, H, W, 3), 77, np.uint8)
    xy, st, dr, bad = _run_chain(make(H, W, h), flat, z, z)
    assert bad == 0 and np.all(st == R.EMPTY) and np.all(dr == 0)

    # capacity below the candidates: the first free slots take the first cells in row-major order, the rest are counted
    full = _run_chain(make(H, W, h), frames[:1], z[:0], z[:0])
    n = int((full[1][0] == R.BORN).sum())
    xy, st, dr, bad = _run_chain(make(H, W, h, max_tracks=5), frames[:1], z[:0], z[:0])
    assert bad == 0 and np.all(st[0] == R.BORN) and dr[0] == n - 5
    assert np.array_equal(xy[0], full[0][0][:5])

    # queries born at frames 0, 5 and 17 (one of them outside the frame) in a 20-frame zero-flow clip
    T2 = 20
    q = np.array([[0, 10.25, 20.5], [5, 63.0, 47.0], [17, 70.0, 3.0], [17, 2.0, 2.0]], np.float32)
    f2, z2 = frames[:1].repeat(T2, 0), np.zeros((T2 - 1, H, W, 2), np.float32)
    xy, st, dr, bad = _run_chain(make(H, W, h, queries=q), f2, z2, z2)
    assert bad == 0
    assert st[0, 0] == R.BORN and np.all(st[1:, 0] == R.TRACKED) and np.all(xy[:, 0] == q[0, 1:])
    assert np.all(st[:5, 1] == R.EMPTY) and st[5, 1] == R.BORN and np.all(st[6:, 1] == R.TRACKED)
    assert np.all(st[:17, 2] == R.EMPTY) and st[17, 2] == R.LEFT and np.all(st[18:, 2] == R.EMPTY)
    assert np.all(np.isnan(xy[17, 2])) and st[17, 3] == R.BORN and np.array_equal(xy[19, 3], q[3, 1:])
    assert np.all(st[:, 4:][st[:, 4:] != R.EMPTY] != R.LEFT)              # the dense slots never see the queries' LEFT


def test_known_answers_on_host(emu):
    _known_answers(lambda H, W, h, **kw: HostTracker(emu, H, W, h, **kw))


class OracleTracker:
    """The oracle as a tracker (the comparisons then hold trivially; used for the scene)."""

    def __init__(self, H, W, spacing=8, tau=0.001, max_tracks=None, queries=None):
        self.H, self.W, self.h, self.tau = H, W, spacing, tau
        self.q = np.zeros((0, 3), np.float32) if queries is None else np.asarray(queries, np.float32)
        self.K = R.capacity(H, W, spacing, max_tracks, queries)
        self.pos, self.status, self.k = np.full((self.K, 2), np.nan, np.float32), np.zeros(self.K, np.uint8), 0

    def texture(self, frame):
        lam = R.texture(frame, self.h)
        return lam, np.array([lam.max(initial=0.0)])

    def advance(self, ffw, fbw):
        a = R.advance(self.pos, self.status, ffw, fbw, **CONSTS)
        self.pos, self.status = a["pos"], a["status"]

    def seed(self, lam, lmax):
        self.pos, self.status, d = R.seed(self.pos, self.status, lam, lmax, self.q, self.k, self.h, self.tau, self.H,
                                          self.W)
        self.k += 1
        return self.pos.copy(), self.status.copy(), d


def test_known_answers_of_the_oracle():
    _known_answers(lambda H, W, h, **kw: OracleTracker(H, W, h, **kw))


# ---------------------------------------------------------------------------------------------------------------
# the synthetic occlusion scene: background moving (2,2) px per frame, a 40 x 40 square (12,6) px per frame
# ---------------------------------------------------------------------------------------------------------------
SCENE_T = 11
DBG, DFG, SQ0 = np.array([2, 2]), np.array([12, 6]), np.array([30, 20])   # (x, y)


def _scene():
    from scipy.ndimage import gaussian_filter
    rng = np.random.default_rng(0)
    H, W = 144, 256
    pad = 2 * SCENE_T + 4

    def tex(h, w, s):
        t = np.stack([gaussian_filter(rng.standard_normal((h, w)), s) for _ in range(3)], -1)
        return np.rint((t - t.min()) / (t.max() - t.min()) * 255).astype(np.uint8)

    bg, fg = tex(H + pad, W + pad, 1.5), tex(40, 40, 1.0)
    frames, sq = [], []
    for k in range(SCENE_T):
        o = k * DBG
        im = bg[pad - o[1]:pad - o[1] + H, pad - o[0]:pad - o[0] + W].copy()
        s = SQ0 + k * DFG
        im[s[1]:s[1] + 40, s[0]:s[0] + 40] = fg
        frames.append(im)
        sq.append(s)
    ffw, fbw = [], []
    for k in range(SCENE_T - 1):
        f = np.broadcast_to(DBG.astype(np.float32), (H, W, 2)).copy()
        f[sq[k][1]:sq[k][1] + 40, sq[k][0]:sq[k][0] + 40] = DFG
        b = np.broadcast_to(-DBG.astype(np.float32), (H, W, 2)).copy()
        b[sq[k + 1][1]:sq[k + 1][1] + 40, sq[k + 1][0]:sq[k + 1][0] + 40] = -DFG
        ffw.append(f)
        fbw.append(b)
    return np.stack(frames), np.stack(ffw), np.stack(fbw), sq


def _in_square(p, s, margin=0):
    return (p[..., 0] >= s[0] + margin) & (p[..., 0] <= s[0] + 39 - margin) & (p[..., 1] >= s[1] + margin) & \
        (p[..., 1] <= s[1] + 39 - margin)


def _check_scene(xy, st):
    frames, ffw, fbw, sq = _scene()
    H, W = frames.shape[1:3]
    occluded = boundary = 0
    for k in range(1, SCENE_T):
        prev_alive = (st[k - 1] == R.TRACKED) | (st[k - 1] == R.BORN)
        p = xy[k - 1]
        n = np.clip(np.rint(np.nan_to_num(p)), 0, [W - 1, H - 1]).astype(int)
        for code in (R.OCCLUDED, R.BOUNDARY):
            ended = prev_alive & (st[k] == code)
            if code == R.OCCLUDED:          # background points the square covers in frame k
                assert np.all(_in_square(p[ended] + DBG, sq[k])), k
                assert np.all(ffw[k - 1][n[ended, 1], n[ended, 0]] == DBG), k
                occluded += int(ended.sum())
            else:                           # points on the square's edge (their flow gradient is not zero)
                e = n[ended]
                near = np.zeros(len(e), bool)
                for dx, dy in ((1, 0), (-1, 0), (0, 1), (0, -1)):
                    a = np.clip(e + [dx, dy], 0, [W - 1, H - 1])
                    near |= np.any(ffw[k - 1][a[:, 1], a[:, 0]] != ffw[k - 1][e[:, 1], e[:, 0]], -1)
                assert np.all(near), k
                boundary += int(ended.sum())
    assert occluded > 0 and boundary > 0, (occluded, boundary)
    # survivors: frame-0 tracks whose true path stays inside the frame and at least 2 px inside the square, or at least
    # 2 px away from it, in every frame, are alive at frame 10 at their exact positions
    born = np.flatnonzero(st[0] == R.BORN)
    survived = 0
    for s in born:
        p0 = xy[0, s]
        fgp = _in_square(p0, sq[0])
        d = DFG if fgp else DBG
        path = p0 + np.arange(SCENE_T)[:, None] * d
        ok = np.all((path >= 0) & (path <= [W - 1, H - 1]))
        for k in range(SCENE_T):
            ok &= bool(_in_square(path[k], sq[k], 2)) if fgp else not _in_square(path[k], sq[k], -3)
        if ok:
            assert np.all(st[1:, s] == R.TRACKED), (s, p0, st[:, s])
            assert np.array_equal(xy[:, s], path.astype(np.float32)), s
            survived += 1
    assert survived >= 20, survived
    return occluded, boundary, survived


def test_synthetic_scene_through_the_oracle():
    frames, ffw, fbw, _ = _scene()
    xy, st, dr = R.track(frames, ffw, fbw, spacing=8)
    print("occluded, boundary, survivors:", _check_scene(xy, st))


def test_synthetic_scene_from_the_host_kernels(emu):
    frames, ffw, fbw, _ = _scene()
    xy, st, dr, bad = _run_chain(HostTracker(emu, frames.shape[1], frames.shape[2], 8), frames, ffw, fbw)
    assert bad == 0
    _check_scene(xy, st)
    ref = R.track(frames, ffw, fbw, spacing=8)
    assert np.array_equal(st, ref[1]) and np.array_equal(np.nan_to_num(xy, nan=-1), np.nan_to_num(ref[0], nan=-1))


# ---------------------------------------------------------------------------------------------------------------
# controls: each changes the rule in one place and must fail the comparison with the kernel
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("control", R.CONTROLS)
def test_controls_fail_the_oracle_comparison(emu, control):
    frames, ffw, fbw, _ = _scene()
    H, W = frames.shape[1:3]
    rng = np.random.default_rng(4)
    sub = (ffw + rng.uniform(-0.4, 0.4, ffw.shape)).astype(np.float32)      # subpixel positions
    bad_ref = _run_chain(HostTracker(emu, H, W, 8), frames[:6], sub[:5], fbw[:5])[3]
    assert bad_ref == 0
    bad = _run_chain(HostTracker(emu, H, W, 8), frames[:6], sub[:5], fbw[:5], control=control)[3]
    print(f"control {control}: {bad} mismatching slots")
    assert bad >= 5, (control, bad)


# ---------------------------------------------------------------------------------------------------------------
# CPU: argument errors and the host bookkeeping
# ---------------------------------------------------------------------------------------------------------------
def test_c_argument_errors_need_no_gpu():
    L = _lib.lib()
    buf = (ctypes.c_double * 64)()
    p = ctypes.cast(buf, ctypes.c_void_p)
    odd = ctypes.c_void_p(p.value + 4)
    assert L.mfn_track_seed_workspace_bytes(10) == 40 and L.mfn_track_seed_workspace_bytes(0) == 0

    def tex(ptrs=None, F=1, H=8, W=8, h=4):
        return L.mfn_track_texture(*(ptrs or [p] * 3), F, H, W, h, None)

    for k in range(3):
        ptrs = [p] * 3
        ptrs[k] = None
        assert tex(ptrs) == -1 and b"null pointer" in L.mfn_last_error(), k
    for F, H, W in ((0, 8, 8), (1, 0, 8), (1, 8, -1)):
        assert tex(F=F, H=H, W=W) == -1 and b"extent" in L.mfn_last_error()
    assert tex(h=0) == -1 and b"spacing" in L.mfn_last_error()
    assert tex([p, odd, p]) == -1 and b"aligned" in L.mfn_last_error()
    assert tex(H=1 << 16, W=1 << 15) == -3 and tex(F=65536) == -3 and b"overflow" in L.mfn_last_error()

    def adv(ptrs=None, K=4, H=8, W=8, h=4, c=(0.01, 0.5, 0.01, 0.002)):
        return L.mfn_track_advance(*(ptrs or [p] * 5), K, H, W, h, *c, None)

    for k in range(5):
        ptrs = [p] * 5
        ptrs[k] = None
        assert adv(ptrs) == -1 and b"null pointer" in L.mfn_last_error(), k
    assert adv(K=0) == -1 and b"extent" in L.mfn_last_error()
    assert adv(h=0) == -1 and b"spacing" in L.mfn_last_error()
    for j in range(4):
        for bad in (-0.1, float("nan"), float("inf")):
            c = [0.01, 0.5, 0.01, 0.002]
            c[j] = bad
            assert adv(c=c) == -1 and b"finite" in L.mfn_last_error(), (j, bad)
    for k in (0, 1, 2):
        ptrs = [p] * 5
        ptrs[k] = odd
        assert adv(ptrs) == -1 and b"aligned" in L.mfn_last_error(), k
    assert adv(H=1 << 16, W=1 << 15) == -3

    def seed(ptrs=None, M=1, nb=64, out=(p, p), K=4, H=8, W=8, h=4, tau=0.001):
        a = ptrs or [p] * 9
        return L.mfn_track_seed(a[0], a[1], a[2], M, a[3], a[4], a[5], a[6], a[7], a[8], nb, out[0], out[1], K, H, W, h,
                                tau, None)

    for k in range(9):
        ptrs = [p] * 9
        ptrs[k] = None
        assert seed(ptrs) == -1 and b"null pointer" in L.mfn_last_error(), k
    ptrs = [p] * 9
    ptrs[2] = None
    # no queries: no query pointer needed.  The short workspace, the last check before the launch, keeps the kernel from
    # running on these host buffers where a GPU is present
    assert seed(ptrs, M=0, nb=15) == -1 and b"workspace" in L.mfn_last_error()
    assert seed(out=(p, None)) == -1 and b"together" in L.mfn_last_error()
    assert seed(K=0, M=0) == -1 and b"extent" in L.mfn_last_error()
    assert seed(h=0) == -1 and b"spacing" in L.mfn_last_error()
    assert seed(M=5) == -1 and b"capacity" in L.mfn_last_error()
    assert seed(M=-1) == -1 and b"capacity" in L.mfn_last_error()
    for tau in (-1.0, float("nan"), float("inf")):
        assert seed(tau=tau) == -1 and b"tau" in L.mfn_last_error(), tau
    for k in (0, 3):
        ptrs = [p] * 9
        ptrs[k] = odd
        assert seed(ptrs) == -1 and b"aligned" in L.mfn_last_error(), k
    assert seed(nb=15) == -1 and b"workspace" in L.mfn_last_error()
    assert seed(H=1 << 16, W=1 << 15) == -3


def test_ops_and_video_argument_errors_need_no_gpu():
    with pytest.raises(MaskflowError, match="spacing"):
        ops.TrackState(8, 8, spacing=0)
    with pytest.raises(MaskflowError, match="tau"):
        ops.TrackState(8, 8, tau=float("nan"))
    with pytest.raises(MaskflowError, match="boundary"):
        ops.TrackState(8, 8, boundary=(0.01, -1.0))
    with pytest.raises(MaskflowError, match="boundary"):
        ops.TrackState(8, 8, boundary=0.01)
    with pytest.raises(MaskflowError, match="queries"):
        ops.TrackState(8, 8, queries=np.zeros((2, 2)))
    with pytest.raises(MaskflowError, match="integer frame"):
        ops.TrackState(8, 8, queries=[[0.5, 1, 1]])
    with pytest.raises(MaskflowError, match="max_tracks"):
        ops.TrackState(8, 8, max_tracks=-1)
    with pytest.raises(MaskflowError, match="slots"):
        ops.TrackState(4, 4, spacing=8)                     # no cell and no query: no slot
    with pytest.raises(MaskflowError, match="CUDA"):
        ops.track_texture(torch.zeros(1, 8, 8, 3, dtype=torch.uint8))
    net = torch.nn.Identity()
    with pytest.raises(MaskflowError, match="spacing"):
        VideoTracker(net, spacing=0)
    with pytest.raises(MaskflowError, match="queries"):
        VideoTracker(net, queries=np.zeros((3,)))
    with pytest.raises(MaskflowError, match="batch"):
        VideoTracker(net, batch=0)
    t = VideoTracker(net, queries=[[0, 1, 2], [3, 4, 5]])
    assert t.bidirectional and t._outputs() == ("xy", "status") and t.num_queries == 2


def _frame(ids, xy, born, eids=(), ereason=()):
    return TrackFrame(np.asarray(ids, np.int64), np.asarray(xy, np.float32).reshape(-1, 2), np.asarray(born, bool),
                      np.asarray(eids, np.int64), np.asarray(ereason, np.uint8))


def test_collect_tracks_on_hand_made_frames():
    frames = [_frame([0, 2, 3], [[1, 1], [5, 5], [7, 7]], [1, 1, 1], [1], [R.LEFT]),
              _frame([0, 3, 4], [[2, 1], [8, 7], [9, 9]], [0, 0, 1], [2], [R.OCCLUDED]),
              _frame([4, 5], [[10, 9], [0, 0]], [0, 1], [0, 3], [R.BOUNDARY, R.LEFT])]
    got = collect_tracks(frames)
    assert np.array_equal(got["start"], [0, 0, 0, 0, 1, 2])
    assert np.array_equal(got["length"], [2, 0, 1, 2, 2, 1])
    assert np.array_equal(got["offset"], [0, 2, 2, 3, 5, 7])
    assert np.array_equal(got["reason"], [R.BOUNDARY, R.LEFT, R.OCCLUDED, R.LEFT, 0, 0])
    assert np.array_equal(got["xy"], np.array([[1, 1], [2, 1], [5, 5], [7, 7], [8, 7], [9, 9], [10, 9], [0, 0]],
                                              np.float32))
    empty = collect_tracks([])
    assert all(len(v) == 0 for v in empty.values())


def test_track_ids_follow_birth_frame_then_slot():
    """Slots 0-1 are queries; dense slots 2-4.  A dense slot stopped in frame 1 is reseeded in frame 2 with a new id."""
    nan = np.nan
    st = np.array([[0, 2, 2, 0, 2], [2, 1, 4, 2, 1], [1, 3, 2, 1, 1]], np.uint8)
    xy = np.zeros((3, 5, 2), np.float32)
    xy[st == 0] = xy[st >= 3] = nan
    fr = list(track_frames(xy, st, num_queries=2))
    assert list(fr[0].ids) == [1, 2, 3] and list(fr[0].born) == [True] * 3
    assert list(fr[1].ids) == [0, 1, 4, 3] and list(fr[1].born) == [True, False, True, False]
    assert list(fr[1].ended_ids) == [2] and list(fr[1].ended_reason) == [R.OCCLUDED]
    assert list(fr[2].ids) == [0, 5, 4, 3] and list(fr[2].ended_ids) == [1] and list(fr[2].ended_reason) == [R.LEFT]


def _cli(name):
    spec = importlib.util.spec_from_file_location(name, os.path.join(ROOT, "tools", name + ".py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_command_line_arguments(tmp_path):
    cli = _cli("track_video")
    a = cli.parse_args(["t.npz", "--video_filepath", "in.mp4", "-c", "w.params"])
    assert (a.spacing, a.queries, a.overlay, a.tail, a.precision, a.batch) == (8, None, None, 15, "fp32", 8)
    qf = tmp_path / "q.csv"
    qf.write_text("t,x,y\n0,1.5,2\n3,4,5.25\n")
    a = cli.parse_args(["t.npz", "--video_filepath", "i.avi", "-c", "w", "--spacing", "4", "--queries", str(qf),
                        "--overlay", "o.avi", "--tail", "5", "--precision", "bf16"])
    assert a.spacing == 4 and a.overlay == "o.avi" and a.tail == 5 and a.precision == "bf16"
    assert np.array_equal(cli.read_queries(str(qf)), np.array([[0, 1.5, 2], [3, 4, 5.25]]))
    for bad in (["t.npz", "-c", "w"], ["t.npz", "--video_filepath", "i", "-c", "w", "--spacing", "0"],
                ["t.npz", "--video_filepath", "i", "-c", "w", "--tail", "0"]):
        with pytest.raises(SystemExit):
            cli.parse_args(bad)


# ---------------------------------------------------------------------------------------------------------------
# GPU: the kernels
# ---------------------------------------------------------------------------------------------------------------
GPU_CASES = [(8, 436, 1024, 8), (8, 436, 1024, 4), (2, 1080, 1920, 8), (2, 1080, 1920, 4)]


@pytest.mark.gpu
@pytest.mark.parametrize("T,H,W,h", GPU_CASES, ids=[f"{t}x{hh}x{w}-s{h}" for t, hh, w, h in GPU_CASES])
def test_kernels_match_oracle(T, H, W, h):
    rng = np.random.default_rng(H + h)
    frames = _textured(rng, T, H, W)
    ffw, fbw = _flows(rng, T, H, W)
    q = np.array([[0, 5.5, 7.25], [1, W - 1, H - 1], [T - 1, -1, 3]], np.float32)
    tally = Tally()
    *_, bad = _run_chain(GpuTracker(H, W, h, queries=q), frames, ffw, fbw, tally)
    assert bad == 0
    tally.check()


@pytest.mark.gpu
def test_known_answers_and_scene_from_the_kernels():
    _known_answers(lambda H, W, h, **kw: GpuTracker(H, W, h, **kw))
    frames, ffw, fbw, _ = _scene()
    xy, st, dr, bad = _run_chain(GpuTracker(frames.shape[1], frames.shape[2], 8), frames, ffw, fbw)
    assert bad == 0
    print("occluded, boundary, survivors:", _check_scene(xy, st))


@pytest.mark.gpu
def test_ops_argument_errors():
    st = ops.TrackState(16, 24, spacing=4)
    f = torch.zeros(16, 24, 2, device="cuda")
    for a, b in ((f.double(), f), (f, f[:8].contiguous()), (f, f.transpose(0, 1).contiguous()), (f.cpu(), f)):
        with pytest.raises(MaskflowError, match="track_advance"):
            ops.track_advance(st, a, b)
    with pytest.raises(MaskflowError, match="forward-only"):
        ops.track_advance(st, f.clone().requires_grad_(), f)
    lam, lmax = ops.track_texture(torch.zeros(16, 24, 3, dtype=torch.uint8, device="cuda"), 4)
    assert lam.shape == (4, 6) and lmax.shape == (1,)
    with pytest.raises(MaskflowError, match="lambda2"):
        ops.track_seed(st, lam[:3].contiguous(), lmax)
    with pytest.raises(MaskflowError, match="out_xy"):
        ops.track_seed(st, lam, lmax, out_xy=torch.empty(3, 2, device="cuda"))


# ---------------------------------------------------------------------------------------------------------------
# GPU: the network and the video tracker
# ---------------------------------------------------------------------------------------------------------------
def _model(cls):
    torch.manual_seed(7)
    return cls().cuda().eval()


def _video(n, H, W, seed):
    """A textured clip moving a few pixels per frame, so the tracks move too."""
    rng = np.random.default_rng(seed)
    big = _textured(rng, 1, H + 4 * n, W + 4 * n)[0]
    return np.stack([big[2 * k:2 * k + H, 3 * k:3 * k + W] for k in range(n)])


def _same_frames(a, b, what):
    assert len(a) == len(b), (what, len(a), len(b))
    for k, (x, y) in enumerate(zip(a, b)):
        for f in TrackFrame._fields:
            assert np.array_equal(getattr(x, f), getattr(y, f), equal_nan=f == "xy"), (what, k, f)


@pytest.mark.gpu
@pytest.mark.parametrize("cls", [network.MaskFlownetS, network.MaskFlownet], ids=["MaskFlownetS", "MaskFlownet"])
def test_video_tracker_equals_track_video(cls):
    """At batch 4: 10 frames (two full batches and a partial one), 3 frames (shorter than one batch), 1 frame, and the
    10-frame video again on the same tracker (the state is reset): every TrackFrame equals, bit for bit, the ones built
    from network.track_video on the device clip."""
    model = _model(cls)
    B, resize, H, W = 4, (128, 192), 100, 150
    q = np.array([[0, 20.5, 30.25], [2, 149, 99], [4, 200, 5]], np.float32)
    with _deterministic():
        tracker = VideoTracker(model, batch=B, resize=resize, spacing=8, queries=q)
        for n, seed in ((10, 1), (3, 2), (1, 3), (10, 1)):
            frames = _video(n, H, W, seed)
            got = list(tracker.run(iter(frames)))
            xy, st, dr = network.track_video(model, torch.from_numpy(frames).cuda(), batch=B, resize=resize, spacing=8,
                                             queries=q)
            want = list(track_frames(xy.cpu().numpy(), st.cpu().numpy(), len(q)))
            _same_frames(got, want, (cls.__name__, n))
            if n == 10:
                assert sum(len(f.ids) for f in got) > 0 and any(len(f.ended_ids) for f in got)


@pytest.mark.gpu
def test_track_video_end_to_end(tmp_path):
    cv2 = pytest.importorskip("cv2")
    cli = _cli("track_video")
    model = _model(network.MaskFlownetS)
    H, W = 96, 128
    frames = _video(6, H, W, seed=6)
    src = str(tmp_path / "in.avi")
    wr = cv2.VideoWriter(src, cv2.VideoWriter_fourcc(*"MJPG"), 10.0, (W, H))
    for f in frames:
        wr.write(f)
    wr.release()
    out, ov = str(tmp_path / "t.npz"), str(tmp_path / "o.avi")
    q = np.array([[0, 10, 10], [2, 50, 40]], np.float32)
    n = cli.track_file(model, out, src, spacing=8, queries=q, overlay=ov, tail=3, batch=4)
    assert n == len(frames)
    z = np.load(out)
    assert set(z.files) >= {"start", "length", "offset", "xy", "reason"}
    assert z["length"].sum() == len(z["xy"]) and z["start"][0] == 0 and z["start"][1] == 2
    cap = cv2.VideoCapture(ov)
    count = 0
    while True:
        ok, fr = cap.read()
        if not ok:
            break
        assert fr.shape == (H, W, 3)
        count += 1
    cap.release()
    assert count == len(frames)
