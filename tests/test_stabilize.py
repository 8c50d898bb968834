"""Video stabilisation: the kernels (csrc/stabilize.cu, ops.affine_motion, ops.warp_frames_affine), the camera path
(maskflownet_b200/camera.py), network.stabilize_video, video.VideoStabilizer and tools/stabilize_video.py.

CPU: the kernel source compiled for the host (tests/host_emu/stabilize_emu.cpp) against the float64 oracle
(oracle/stabilize_ref.py); known answers, the robustness scene, five controls that must fail the comparison, the camera
path against the oracle, the jitter of a shaky synthetic clip through the oracle, and argument errors.  GPU: the same
through the ops at the video sizes, reproducibility and graph replay, VideoStabilizer bit for bit against
network.stabilize_video, bf16 and the command line.

Tolerances.  The fit is compared as its map applied to the four frame corners, within 1e-6 px: the kernel's sums run in
another order than numpy's, which moves the result by float64 rounding only.  The residual is float32 of a float64 value:
within 1e-5 px plus one float32 ulp of the value, NaN in the same places.  The warp evaluates the oracle's expression in
the same order; the kernel's fused multiply-adds may move a value across a rounding tie, so values may differ by 1, and at
least 99.9 % must be exact.
"""
import ctypes
import importlib.util
import os

import numpy as np
import pytest
import torch

from maskflownet_b200 import MaskflowError, _lib, camera, network, ops
from maskflownet_b200.video import VideoFlowPredictor, VideoStabilizer
from oracle import stabilize_ref as R

from launchcheck.emu import build, ptr
from launchcheck.inputs import _deterministic
from launchcheck.stabilize import CORNER_TOL, WARP_EXACT, _check_fit, _check_warp, _fit_mismatch, _warp_mismatch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


# ---------------------------------------------------------------------------------------------------------------
# inputs
# ---------------------------------------------------------------------------------------------------------------
def _affine_flow(A, H, W):
    y, x = np.mgrid[0:H, 0:W].astype(np.float64)
    return np.stack([A[0, 0] * x + A[0, 1] * y + A[0, 2] - x, A[1, 0] * x + A[1, 1] * y + A[1, 2] - y], -1)


def _rot(deg, scale, cx, cy, tx=0.0, ty=0.0):
    """Rotation by deg with scale about (cx, cy), then a translation."""
    c, s = scale * np.cos(np.radians(deg)), scale * np.sin(np.radians(deg))
    L = np.array([[c, -s], [s, c]])
    t = np.array([cx, cy]) - L @ np.array([cx, cy]) + np.array([tx, ty])
    return np.concatenate([L, t[:, None]], 1)


def _case(rng, N, H, W):
    """Flows of a random camera motion with noise, a moving block, targets outside the frame, and NaN / +-inf."""
    out = np.empty((N, H, W, 2), np.float32)
    for n in range(N):
        A = _rot(rng.uniform(-3, 3), rng.uniform(0.97, 1.03), rng.uniform(0, W - 1), rng.uniform(0, H - 1),
                 rng.uniform(-0.05, 0.05) * W, rng.uniform(-0.05, 0.05) * H)
        f = _affine_flow(A, H, W) + rng.normal(0, 0.4, (H, W, 2))
        y0, x0 = rng.integers(0, H), rng.integers(0, W)
        f[y0:y0 + max(1, H // 4), x0:x0 + max(1, W // 4)] += rng.uniform(-8, 8, 2)
        m = rng.random((H, W)) < 0.03
        f[m] = rng.normal(0, max(H, W), (int(m.sum()), 2))                # anywhere, often outside
        m = rng.random((H, W, 2)) < 0.01
        f[m] = rng.choice([np.nan, np.inf, -np.inf], int(m.sum()))
        out[n] = f
    return out


def _frames(rng, N, H, W):
    """Smooth-ish textured frames (a random image blurred a little), so a bilinear warp has structure to sample."""
    img = rng.integers(0, 256, (N, H + 2, W + 2, 3)).astype(np.float64)
    img = (img[:, :-2, :-2] + img[:, 2:, 2:] + img[:, 1:-1, 1:-1] * 2) / 4
    return np.clip(np.rint(img), 0, 255).astype(np.uint8)


def _matrices(rng, N, H, W):
    return np.stack([_rot(rng.uniform(-10, 10), rng.uniform(0.8, 1.25), rng.uniform(0, W), rng.uniform(0, H),
                          rng.uniform(-0.2, 0.2) * W, rng.uniform(-0.2, 0.2) * H) for _ in range(N)])


HOST_SHAPES = [(2, 37, 53), (1, 1, 40), (1, 40, 1), (2, 64, 96), (1, 3, 3)]


# ---------------------------------------------------------------------------------------------------------------
# the host build
# ---------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    L = build(tmp_path_factory, "stabilize_emu")
    v, i = ctypes.c_void_p, ctypes.c_int
    L.emu_affine_motion.argtypes = [v] * 4 + [i] * 4 + [ctypes.c_float]
    L.emu_warp_frames_affine.argtypes = [v] * 3 + [i] * 3
    L.emu_fit_ctas.argtypes = [i, i]
    return L


def _host_ops(L):
    def fit(flow, iterations=ops.AFFINE_ITERATIONS, sigma=ops.AFFINE_SIGMA):
        flow = np.ascontiguousarray(flow, np.float32)
        N, H, W, _ = flow.shape
        A = np.zeros((N, 2, 3))
        ok = np.zeros(N, np.uint8)
        res = np.zeros((N, H, W), np.float32)
        L.emu_affine_motion(ptr(flow), ptr(A), ptr(ok), ptr(res), N, H, W, iterations, sigma)
        return A, ok.astype(bool), res

    def warp(src, M):
        src = np.ascontiguousarray(src, np.uint8)
        M = np.ascontiguousarray(M, np.float64)
        out = np.zeros_like(src)
        L.emu_warp_frames_affine(ptr(src), ptr(M), ptr(out), *src.shape[:3])
        return out

    return fit, warp


def _gpu_ops():
    def fit(flow, iterations=ops.AFFINE_ITERATIONS, sigma=ops.AFFINE_SIGMA):
        A, ok, res = ops.affine_motion(torch.from_numpy(np.ascontiguousarray(flow, np.float32)).cuda(), iterations, sigma,
                                       want_residual=True)
        return A.cpu().numpy(), ok.cpu().numpy(), res.cpu().numpy()

    def warp(src, M):
        return ops.warp_frames_affine(torch.from_numpy(np.ascontiguousarray(src)).cuda(),
                                      torch.from_numpy(np.ascontiguousarray(M, np.float64)).cuda()).cpu().numpy()

    return fit, warp


# ---------------------------------------------------------------------------------------------------------------
# shared checks, run from the host build and from the GPU
# ---------------------------------------------------------------------------------------------------------------
def _against_oracle(fit, warp, N, H, W, seed):
    rng = np.random.default_rng(seed)
    flow = _case(rng, N, H, W)
    d = _check_fit(fit(flow), R.fit(flow), H, W, f"fit {N}x{H}x{W}")
    src, M = _frames(rng, N, H, W), _matrices(rng, N, H, W)
    e = _check_warp(warp(src, M), R.warp(src, M), f"warp {N}x{H}x{W}")
    return d, e


def _known_answers(fit, warp):
    I = np.eye(2, 3)
    H, W = 48, 80
    A, ok, res = fit(np.zeros((1, H, W, 2), np.float32))
    assert ok.all() and np.abs(A - I).max() <= 1e-12 and np.nanmax(res) <= 1e-9
    T = np.array([[1, 0, 2.5], [0, 1, -1.25]])                       # dyadic translation
    A, ok, _ = fit(_affine_flow(T, H, W).astype(np.float32)[None])
    assert ok.all() and np.abs(R.corners(A, H, W) - R.corners(T, H, W)).max() <= 1e-9
    S = _rot(4.0, 1.05, 11.0, 30.0, 0.7, -0.4)                        # rotation with scale about an off-centre point
    A, ok, _ = fit(_affine_flow(S, H, W).astype(np.float32)[None])
    assert ok.all() and np.abs(R.corners(A, H, W) - R.corners(S, H, W)).max() <= 1e-4
    singular = [np.full((1, H, W, 2), np.nan, np.float32),           # all NaN
                np.full((1, H, W, 2), 2.0 * max(H, W), np.float32),  # every target outside the frame
                _affine_flow(T, 1, W).astype(np.float32)[None]]      # H = 1: the points lie on one line
    for f in singular:
        A, ok, res = fit(f)
        assert not ok.any() and np.array_equal(A, I[None]), A
    rng = np.random.default_rng(3)
    src = _frames(rng, 2, H, W)
    assert np.array_equal(warp(src, np.stack([I, I])), src)
    sh = np.stack([[[1, 0, 3], [0, 1, -2]], [[1, 0, -5], [0, 1, 4]]]).astype(np.float64)   # source = output + (3, -2)
    got = warp(src, sh)
    for n in range(2):
        xs = np.clip(np.arange(W) + int(sh[n, 0, 2]), 0, W - 1)
        ys = np.clip(np.arange(H) + int(sh[n, 1, 2]), 0, H - 1)
        assert np.array_equal(got[n], src[n][np.ix_(ys, xs)]), n


def _robust_scene(seed=0, H=120, W=160):
    """A known camera map, 0.3 px noise, a square over 30 % of the frame moving differently, and NaN holes.  Returns
    (flow (1,H,W,2), the true map, the square's mask, its relative motion in px)."""
    rng = np.random.default_rng(seed)
    A = _rot(1.5, 1.02, 0.4 * W, 0.6 * H, 2.25, -1.5)
    f = _affine_flow(A, H, W) + rng.normal(0, 0.3, (H, W, 2))
    side = int(round(np.sqrt(0.3 * H * W)))
    sq = np.zeros((H, W), bool)
    sq[10:10 + side, 20:20 + side] = True
    rel = np.array([12.0, -8.0])
    f[sq] += rel
    holes = np.zeros((H, W), bool)
    holes[60:70, 5:15] = holes[100:104, 130:150] = True
    f[holes] = np.nan
    return f.astype(np.float32)[None], A, sq & ~holes, float(np.hypot(*rel))


def _robustness(fit):
    flow, A, sq, rel = _robust_scene()
    H, W = flow.shape[1:3]
    got, ok, res = fit(flow)
    err = float(np.abs(R.corners(got, H, W) - R.corners(A, H, W)).max())
    assert ok.all() and err <= 0.06, err
    r = res[0][sq]
    r = r[np.isfinite(r)]                      # the square's pixels whose target stays in the frame
    assert r.size > 0.2 * H * W
    assert abs(float(np.median(r)) - rel) <= 0.1 and np.quantile(r, 0.99) <= rel + 1.2 and r.min() >= rel - 1.2, \
        (np.median(r), r.min(), r.max())
    ls, _, _ = fit(flow, iterations=1)
    miss = float(np.abs(R.corners(ls, H, W) - R.corners(A, H, W)).max())
    assert miss > 1.0, miss
    return err, miss


def _controls_fail(fit, warp):
    rng = np.random.default_rng(11)
    H, W = 45, 70
    flow = _case(rng, 2, H, W)
    got = fit(flow)
    src, M = _frames(rng, 2, H, W), _matrices(rng, 2, H, W)
    wgot = warp(src, M)
    out = {}
    for c in R.CONTROLS:
        if c in R.FIT_CONTROLS:
            d, okbad, resbad = _fit_mismatch(got, R.fit(flow, control=c), H, W)
            out[c] = d > CORNER_TOL or okbad or resbad > 0
        else:
            dmax, exact = _warp_mismatch(wgot, R.warp(src, M, control=c))
            out[c] = dmax > 1 or exact < WARP_EXACT
    assert all(out.values()), out
    # and the comparisons pass without a control
    _check_fit(got, R.fit(flow), H, W)
    _check_warp(wgot, R.warp(src, M))


# ---------------------------------------------------------------------------------------------------------------
# CPU: the host build
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N,H,W", HOST_SHAPES, ids=[f"{n}x{h}x{w}" for n, h, w in HOST_SHAPES])
def test_kernel_source_matches_oracle_on_host(emu, N, H, W):
    fit, warp = _host_ops(emu)
    d, e = _against_oracle(fit, warp, N, H, W, seed=H * W)
    print(f"{N}x{H}x{W}: corners within {d:.2e} px, warp {100 * e:.3f} % exact")


def test_ctas_depend_on_the_frame_size_only(emu):
    assert [emu.emu_fit_ctas(h, w) for h, w in ((1, 1), (1, 2048), (1, 2049), (436, 1024), (1080, 1920))] == \
        [1, 1, 2, 218, 256]


def test_known_answers_on_host(emu):
    _known_answers(*_host_ops(emu))


def test_robustness_on_host(emu):
    err, miss = _robustness(_host_ops(emu)[0])
    print(f"robust fit within {err:.4f} px at the corners; plain least squares misses by {miss:.2f} px")


def test_controls_fail_the_oracle_comparison_on_host(emu):
    _controls_fail(*_host_ops(emu))


def test_robustness_through_the_oracle():
    _robustness(lambda f, iterations=ops.AFFINE_ITERATIONS: R.fit(f, iterations))


# ---------------------------------------------------------------------------------------------------------------
# CPU: the camera path
# ---------------------------------------------------------------------------------------------------------------
def test_camera_path_matches_oracle():
    rng = np.random.default_rng(5)
    H, W = 90, 160
    for T, radius, crop in ((20, 15, 0.9), (7, 2, 1.0), (2, 0, 0.5), (30, 4, 0.8)):
        aff = np.stack([_rot(rng.uniform(-1, 1), rng.uniform(0.99, 1.01), W / 2, H / 2, *rng.uniform(-3, 3, 2))
                        for _ in range(T - 1)])
        ok = rng.random(T - 1) > 0.2
        got = camera.camera_path(aff, ok, H, W, radius, crop)
        assert got.shape == (T, 2, 3)
        assert np.abs(got - R.path(aff, ok, H, W, radius, crop)).max() <= 1e-9


def test_failed_fits_count_as_no_motion():
    rng = np.random.default_rng(6)
    H, W = 40, 60
    aff = np.stack([_rot(0, 1, 0, 0, *rng.uniform(-3, 3, 2)) for _ in range(9)])
    ok = np.ones(9, bool)
    ok[4] = False
    junk = aff.copy()
    junk[4] = np.nan                                 # whatever a failed fit holds, it is not used
    a = camera.camera_path(junk, ok, H, W, 3, 0.9)
    aff_id = aff.copy()
    aff_id[4] = np.eye(2, 3)
    assert np.array_equal(a, camera.camera_path(aff_id, np.ones(9, bool), H, W, 3, 0.9))


def test_constant_pan_and_radius_zero_give_the_zoom():
    H, W, T, R_ = 72, 128, 40, 6
    Z = camera.zoom(H, W, 0.9)[:2]
    pan = np.repeat(np.array([[[1, 0, 1.75], [0, 1, -0.5]]]), T - 1, 0)
    M = camera.camera_path(pan, np.ones(T - 1, bool), H, W, R_, 0.9)
    assert np.abs(M[R_:T - R_] - Z).max() <= 1e-9
    assert np.abs(M[:R_] - Z).max() > 1e-3                   # at the ends the window is one-sided
    rng = np.random.default_rng(2)
    shaky = np.stack([_rot(rng.uniform(-1, 1), 1.0, W / 2, H / 2, *rng.uniform(-3, 3, 2)) for _ in range(T - 1)])
    assert np.array_equal(camera.camera_path(shaky, np.ones(T - 1, bool), H, W, 0, 0.9), np.broadcast_to(Z, (T, 2, 3)))
    assert np.abs(R.path(shaky, np.ones(T - 1, bool), H, W, 0, 0.9) - Z).max() <= 1e-9


def test_windowed_path_equals_the_whole_path():
    """stabilize_path from only the window of P gives the same bits as from the whole path (what the streamer does)."""
    rng = np.random.default_rng(9)
    H, W, T, R_ = 50, 70, 25, 4
    aff = np.stack([_rot(rng.uniform(-1, 1), 1.0, W / 2, H / 2, *rng.uniform(-3, 3, 2)) for _ in range(T - 1)])
    P = [np.eye(3)]
    for a in aff:
        P.append(camera.path_step(P[-1], a, True))
    whole = camera.camera_path(aff, np.ones(T - 1, bool), H, W, R_, 0.9)
    for t in range(T):
        lo = max(0, t - R_)
        win = P[lo:min(T, t + R_ + 1)]
        assert np.array_equal(camera.stabilize_path(win, t, T, H, W, R_, 0.9, first=lo), whole[t]), t
    with pytest.raises(MaskflowError, match="needs"):
        camera.stabilize_path(P[5:], 3, T, H, W, R_, 0.9, first=5)


def _shaky_clip(T=40, H=96, W=128, seed=4):
    """A textured canvas seen by a camera with a smooth pan plus seeded jitter of +-3 px and +-0.5 deg.  G_t maps a
    frame-t pixel to the canvas.  Returns (frames (T,H,W,3), G (T,3,3), the true pair maps (T-1,2,3), true flows)."""
    rng = np.random.default_rng(seed)
    ch, cw = H + 120, W + 3 * T + 120
    canvas = rng.integers(0, 256, (ch // 4 + 2, cw // 4 + 2, 3)).astype(np.float64)
    canvas = np.kron(canvas, np.ones((4, 4, 1)))[:ch, :cw]                    # blocky texture
    G = []
    for t in range(T):
        ang = np.radians(rng.uniform(-0.5, 0.5))
        jx, jy = rng.uniform(-3, 3, 2)
        c, s = np.cos(ang), np.sin(ang)
        L = np.array([[c, -s], [s, c]])
        ctr = np.array([(W - 1) / 2, (H - 1) / 2])
        t_ = np.array([60 + 3.0 * t + jx, 60 + 0.5 * t + jy]) + ctr - L @ ctr
        g = np.eye(3)
        g[:2, :2], g[:2, 2] = L, t_
        G.append(g)
    G = np.stack(G)
    y, x = np.mgrid[0:H, 0:W].astype(np.float64)
    frames = np.empty((T, H, W, 3), np.uint8)
    for t in range(T):
        cx = G[t, 0, 0] * x + G[t, 0, 1] * y + G[t, 0, 2]
        cy = G[t, 1, 0] * x + G[t, 1, 1] * y + G[t, 1, 2]
        x0, y0 = np.floor(cx).astype(int), np.floor(cy).astype(int)
        wx, wy = (cx - x0)[..., None], (cy - y0)[..., None]
        v = ((1 - wy) * ((1 - wx) * canvas[y0, x0] + wx * canvas[y0, x0 + 1])
             + wy * ((1 - wx) * canvas[y0 + 1, x0] + wx * canvas[y0 + 1, x0 + 1]))
        frames[t] = np.clip(np.rint(v), 0, 255).astype(np.uint8)
    A = np.stack([(np.linalg.inv(G[t + 1]) @ G[t])[:2] for t in range(T - 1)])
    flows = np.stack([_affine_flow(a, H, W) for a in A]).astype(np.float32)
    return frames, G, A, flows


def _jitter(V, H, W):
    """Mean |second difference| of the virtual camera's view of the frame centre, V (T,3,3) output -> canvas."""
    c = np.array([(W - 1) / 2, (H - 1) / 2, 1.0])
    p = (V @ c)[:, :2]
    return float(np.linalg.norm(p[2:] - 2 * p[1:-1] + p[:-2], axis=1).mean())


def _jitter_reduction(fit, warp):
    frames, G, A_true, flows = _shaky_clip()
    T, H, W, _ = frames.shape
    A, ok, _ = fit(flows)
    assert ok.all() and np.abs(R.corners(A, H, W) - R.corners(A_true, H, W)).max() <= 1e-3
    M = R.path(A, ok, H, W, 15, 0.9)
    out = warp(frames, M)
    assert out.shape == frames.shape
    V = np.einsum("tij,tjk->tik", G, np.concatenate([M, np.broadcast_to([[[0, 0, 1]]], (T, 1, 3))], 1))
    before, after = _jitter(G, H, W), _jitter(V, H, W)
    return before, after


def test_shaky_clip_jitter_falls_through_the_oracle():
    before, after = _jitter_reduction(R.fit, R.warp)
    print(f"jitter of the frame centre: {before:.3f} -> {after:.3f} px per frame^2, a factor of {before / after:.1f}")
    assert before >= 5 * after, (before, after)


# ---------------------------------------------------------------------------------------------------------------
# CPU: argument errors
# ---------------------------------------------------------------------------------------------------------------
def test_c_argument_errors_need_no_gpu():
    L = _lib.lib()
    buf = (ctypes.c_double * 256)()
    p = ctypes.cast(buf, ctypes.c_void_p)
    odd = ctypes.c_void_p(p.value + 4)
    ws = L.mfn_affine_motion_workspace_bytes
    assert ws(2, 436, 1024) == 8 * 12 * 2 * 218 and ws(1, 1, 1) == 8 * 12 and ws(0, 3, 5) == 0
    f = L.mfn_affine_motion

    def call(*, ptrs=None, nb=2048, N=1, H=2, W=2, it=8, sigma=1.0):
        ptrs = ptrs or [p] * 5
        return f(*ptrs, nb, N, H, W, it, sigma, None)

    for k in (0, 1, 2, 4):
        ptrs = [p] * 5
        ptrs[k] = None
        assert call(ptrs=ptrs) == -1 and b"null pointer" in L.mfn_last_error(), k
    for N, H, W in ((0, 2, 2), (1, 0, 2), (1, 2, -1)):
        assert call(N=N, H=H, W=W) == -1 and b"extent" in L.mfn_last_error()
    assert call(it=0) == -1 and b"iterations" in L.mfn_last_error()
    for s in (0.0, -1.0, float("nan"), float("inf")):
        assert call(sigma=s) == -1 and b"sigma" in L.mfn_last_error(), s
    for k in (0, 1, 4):
        ptrs = [p] * 5
        ptrs[k] = odd
        assert call(ptrs=ptrs) == -1 and b"aligned" in L.mfn_last_error(), k
    assert call(ptrs=[p, p, p, ctypes.c_void_p(p.value + 2), p]) == -1 and b"aligned" in L.mfn_last_error()
    assert call(nb=8 * 12 - 1) == -1 and b"workspace" in L.mfn_last_error()
    assert call(H=1 << 16, W=1 << 15, nb=1 << 30) == -3 and b"overflow" in L.mfn_last_error()
    assert call(N=65536, nb=1 << 30) == -3 and b"overflow" in L.mfn_last_error()
    g = L.mfn_warp_frames_affine
    for k in range(3):
        ptrs = [p] * 3
        ptrs[k] = None
        assert g(*ptrs, 1, 2, 2, None) == -1 and b"null pointer" in L.mfn_last_error(), k
    for N, H, W in ((0, 2, 2), (1, 0, 2), (1, 2, -1)):
        assert g(p, p, p, N, H, W, None) == -1 and b"extent" in L.mfn_last_error()
    assert g(p, odd, p, 1, 2, 2, None) == -1 and b"aligned" in L.mfn_last_error()
    assert g(p, p, p, 1, 1 << 16, 1 << 15, None) == -3 and b"overflow" in L.mfn_last_error()
    assert g(p, p, p, 65536, 2, 2, None) == -3 and b"overflow" in L.mfn_last_error()


def test_ops_path_and_video_argument_errors_need_no_gpu():
    flow = torch.zeros(1, 4, 4, 2)
    for it in (0, -1, 1.5, True):
        with pytest.raises(MaskflowError, match="iterations"):
            ops.affine_motion(flow, iterations=it)
    for s in (0.0, -1.0, float("nan"), float("inf"), "x"):
        with pytest.raises(MaskflowError, match="sigma"):
            ops.affine_motion(flow, sigma=s)
    with pytest.raises(MaskflowError, match="CUDA"):
        ops.affine_motion(flow)
    with pytest.raises(MaskflowError, match="CUDA"):
        ops.warp_frames_affine(torch.zeros(1, 4, 4, 3, dtype=torch.uint8), torch.zeros(1, 2, 3, dtype=torch.float64))
    for bad in (-1, 1.5, True, "3"):
        with pytest.raises(MaskflowError, match="radius"):
            camera.camera_path(np.zeros((2, 2, 3)), np.ones(2, bool), 4, 4, radius=bad)
    for bad in (0.0, -0.5, 1.01, float("nan"), "x"):
        with pytest.raises(MaskflowError, match="crop"):
            camera.camera_path(np.zeros((2, 2, 3)), np.ones(2, bool), 4, 4, crop=bad)
    with pytest.raises(MaskflowError, match="ok flags"):
        camera.camera_path(np.zeros((2, 2, 3)), np.ones(3, bool), 4, 4)
    net = torch.nn.Identity()
    for kw, msg in ((dict(radius=-1), "radius"), (dict(crop=0.0), "crop"), (dict(crop=1.5), "crop"),
                    (dict(iterations=0), "iterations"), (dict(sigma=0.0), "sigma"), (dict(sigma=float("inf")), "sigma"),
                    (dict(batch=0), "batch")):
        with pytest.raises(MaskflowError, match=msg):
            VideoStabilizer(net, **kw)
    s = VideoStabilizer(net, batch=4, radius=5)
    assert s._outputs() == ("affine", "ok") and not s.bidirectional and s.ring_size == 5 + 2 * 4 + 1
    assert s._segments(12, 17) == [(12, 14), (14, 17)] and s._segments(0, 3) == [(0, 3)]
    with pytest.raises(MaskflowError, match="clip"):
        network.stabilize_video(net, torch.zeros(3, 4, 4, 3))
    with pytest.raises(MaskflowError, match="radius"):
        network.stabilize_video(net, torch.zeros(3, 4, 4, 3, dtype=torch.uint8), radius=-2)


def _cli():
    spec = importlib.util.spec_from_file_location("stabilize_video", os.path.join(ROOT, "tools", "stabilize_video.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_command_line_arguments():
    cli = _cli()
    a = cli.parse_args(["out.mp4", "--video_filepath", "in.mp4", "-c", "w.params"])
    assert (a.radius, a.crop, a.batch, a.resize, a.precision, a.network) == (15, 0.9, 8, None, "fp32", "MaskFlownet")
    a = cli.parse_args(["o.avi", "--video_filepath", "i.avi", "-c", "w.pt", "-n", "MaskFlownet_S", "--radius", "0",
                        "--crop", "1", "--batch", "3", "--resize", "448,1024", "--precision", "bf16"])
    assert (a.radius, a.crop, a.batch, a.resize, a.precision, a.network) == (0, 1.0, 3, (448, 1024), "bf16",
                                                                            "MaskFlownet_S")
    for bad in (["o.mp4", "-c", "w"],
                ["o.mp4", "--video_filepath", "i.mp4"],
                ["o.mp4", "--video_filepath", "i.mp4", "-c", "w", "--radius", "-1"],
                ["o.mp4", "--video_filepath", "i.mp4", "-c", "w", "--crop", "0"],
                ["o.mp4", "--video_filepath", "i.mp4", "-c", "w", "--crop", "1.2"],
                ["o.mp4", "--video_filepath", "i.mp4", "-c", "w", "--batch", "0"],
                ["o.mp4", "--video_filepath", "i.mp4", "-c", "w", "--resize", "448"]):
        with pytest.raises(SystemExit):
            cli.parse_args(bad)


# ---------------------------------------------------------------------------------------------------------------
# GPU: the kernels
# ---------------------------------------------------------------------------------------------------------------
GPU_SHAPES = [(8, 436, 1024), (2, 1080, 1920), (3, 37, 53), (1, 1, 257), (1, 257, 1)]


@pytest.mark.gpu
@pytest.mark.parametrize("N,H,W", GPU_SHAPES, ids=[f"{n}x{h}x{w}" for n, h, w in GPU_SHAPES])
def test_kernels_match_oracle(N, H, W):
    d, e = _against_oracle(*_gpu_ops(), N, H, W, seed=H + W)
    print(f"{N}x{H}x{W}: corners within {d:.2e} px, warp {100 * e:.3f} % exact")


@pytest.mark.gpu
def test_known_answers_robustness_and_controls_on_gpu():
    fit, warp = _gpu_ops()
    _known_answers(fit, warp)
    err, miss = _robustness(fit)
    print(f"robust fit within {err:.4f} px at the corners; plain least squares misses by {miss:.2f} px")
    _controls_fail(fit, warp)
    before, after = _jitter_reduction(fit, warp)
    print(f"jitter from the kernels: {before:.3f} -> {after:.3f}, a factor of {before / after:.1f}")
    assert before >= 5 * after


@pytest.mark.gpu
def test_reproducible_batch_independent_and_graph_replay():
    rng = np.random.default_rng(1)
    flow = torch.from_numpy(_case(rng, 8, 436, 1024)).cuda()
    src = torch.from_numpy(_frames(rng, 8, 436, 1024)).cuda()
    M = torch.from_numpy(_matrices(rng, 8, 436, 1024)).cuda()
    a1, ok1, r1 = ops.affine_motion(flow, want_residual=True)
    a2, ok2, r2 = ops.affine_motion(flow, want_residual=True)
    assert torch.equal(a1, a2) and torch.equal(ok1, ok2) and torch.equal(r1.isnan(), r2.isnan())
    assert torch.equal(r1.nan_to_num(), r2.nan_to_num())
    a3, _ = ops.affine_motion(flow[5:6].contiguous())
    assert torch.equal(a3[0], a1[5])
    w1 = ops.warp_frames_affine(src, M)
    assert torch.equal(w1, ops.warp_frames_affine(src, M))
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ops.affine_motion(flow, want_residual=True)
        ops.warp_frames_affine(src, M)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        ga, gok, gr = ops.affine_motion(flow, want_residual=True)
        gw = ops.warp_frames_affine(src, M)
    for v in (ga, gr, gw):
        v.zero_()
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(ga, a1) and torch.equal(gok, ok1) and torch.equal(gw, w1)
    assert torch.equal(gr.nan_to_num(), r1.nan_to_num()) and torch.equal(gr.isnan(), r1.isnan())


@pytest.mark.gpu
def test_ops_argument_errors():
    flow = torch.zeros(2, 8, 8, 2, device="cuda")
    for bad in (flow.double(), flow.transpose(1, 2), flow[..., :1].contiguous(), flow[0]):
        with pytest.raises(MaskflowError, match="affine_motion"):
            ops.affine_motion(bad)
    with pytest.raises(MaskflowError, match="forward-only"):
        ops.affine_motion(flow.clone().requires_grad_())
    fr = torch.zeros(2, 8, 8, 3, dtype=torch.uint8, device="cuda")
    M = torch.zeros(2, 2, 3, dtype=torch.float64, device="cuda")
    for bf, bm in ((fr.float(), M), (fr[..., :2].contiguous(), M), (fr.transpose(1, 2), M), (fr, M.float()),
                   (fr, M[:1]), (fr, M.cpu()), (fr, M.transpose(1, 2).contiguous())):
        with pytest.raises(MaskflowError, match="warp_frames_affine"):
            ops.warp_frames_affine(bf, bm)


# ---------------------------------------------------------------------------------------------------------------
# GPU: the network and the video stabiliser
# ---------------------------------------------------------------------------------------------------------------
def _model(cls):
    torch.manual_seed(7)
    return cls().cuda().eval()


def _video(n, H, W, seed):
    return _frames(np.random.default_rng(seed), n, H, W)


def _stream_equals_eager(stab, model, clip, what):
    got = list(stab.run(iter(clip)))
    assert len(got) == len(clip), (what, len(got))
    want, aff, ok, M = network.stabilize_video(model, torch.from_numpy(clip).cuda(), batch=stab.batch,
                                               resize=stab.resize, radius=stab.radius, crop=stab.crop)
    assert aff.shape == (len(clip) - 1, 2, 3) and ok.shape == (len(clip) - 1,) and M.shape == (len(clip), 2, 3)
    want = want.cpu().numpy()
    for t, fr in enumerate(got):
        assert fr.shape == clip.shape[1:] and fr.dtype == np.uint8
        assert np.array_equal(fr, want[t]), (what, t)


@pytest.mark.gpu
@pytest.mark.parametrize("cls", [network.MaskFlownetS, network.MaskFlownet], ids=lambda c: c.__name__)
def test_video_stabilizer_equals_eager_chain(cls):
    """Batch 4: a 10-frame video (two full batches and one of one pair), run twice on the same stabiliser, then 3, 2 and 1
    frames; radius 0 and a radius longer than the video."""
    model = _model(cls)
    H, W, resize = 100, 150, (128, 192)
    with _deterministic():
        stab = VideoStabilizer(model, batch=4, resize=resize, radius=3)
        clip = _video(10, H, W, seed=1)
        _stream_equals_eager(stab, model, clip, "10 frames")
        _stream_equals_eager(stab, model, clip, "10 frames again")
        for n in (3, 2, 1):
            _stream_equals_eager(stab, model, _video(n, H, W, seed=n), f"{n} frames")
        for radius in (0, 25):
            _stream_equals_eager(VideoStabilizer(model, batch=4, resize=resize, radius=radius), model, clip,
                                 f"radius {radius}")


@pytest.mark.gpu
def test_failed_fit_is_identity_in_the_eager_chain():
    """A clip of flat frames gives zero flow everywhere except where the random network says otherwise; a pair with an
    H = 1 frame cannot be fitted at all: ok is False and the fit is the identity."""
    model = _model(network.MaskFlownetS)
    clip = torch.from_numpy(_video(3, 1, 64, seed=2)).cuda()
    out, aff, ok, M = network.stabilize_video(model, clip, batch=2, radius=2, crop=1.0)
    assert not ok.any() and torch.equal(aff.cpu(), torch.eye(2, 3, dtype=torch.float64).expand(2, 2, 3))
    assert np.abs(M - np.eye(2, 3)).max() <= 1e-12 and torch.equal(out, clip)


@pytest.mark.gpu
def test_bf16_mode_and_video_predictor_unchanged():
    model = _model(network.MaskFlownetS)
    model.inference_precision = "bf16"
    clip = _video(6, 96, 128, seed=3)
    with _deterministic():
        _stream_equals_eager(VideoStabilizer(model, batch=4, radius=2), model, clip, "bf16")
    model.inference_precision = "fp32"
    got = list(VideoFlowPredictor(model, batch=4).run(iter(clip)))
    assert len(got) == len(clip) - 1 and got[0].shape == (96, 128, 3)


@pytest.mark.gpu
def test_stabilize_video_end_to_end(tmp_path):
    cv2 = pytest.importorskip("cv2")
    cli = _cli()
    model = _model(network.MaskFlownetS)
    H, W = 64, 96
    frames = _video(7, H, W, seed=6)
    src = str(tmp_path / "in.avi")
    wr = cv2.VideoWriter(src, cv2.VideoWriter_fourcc(*"MJPG"), 12.0, (W, H))
    for f in frames:
        wr.write(f)
    wr.release()
    dst = str(tmp_path / "out.avi")
    n, fps = cli.stabilize_file(model, dst, src, radius=2, crop=0.9, batch=4)
    assert n == len(frames) and fps == pytest.approx(12.0)
    cap = cv2.VideoCapture(dst)
    assert cap.get(cv2.CAP_PROP_FPS) == pytest.approx(12.0)
    count = 0
    while True:
        ok, fr = cap.read()
        if not ok:
            break
        assert fr.shape == (H, W, 3)
        count += 1
    cap.release()
    assert count == len(frames)
