"""Moving-object segmentation: the kernels (csrc/motionseg.cu, ops.segment_motion), network.segment_motion,
video.VideoMotionSegmenter and tools/segment_video.py.

CPU: the oracle's labelling (oracle/motionseg_ref.py) against scipy.ndimage.label; the kernel source compiled for the host
(tests/host_emu/motionseg_emu.cpp) against the oracle on shapes and masks chosen to be hard for a union-find, with the
unions in shuffled orders; two controls that must fail the comparison; the synthetic scene through the oracle; argument
errors and the command line.  GPU: the same through the ops at the video sizes, reproducibility and graph replay,
VideoMotionSegmenter bit for bit against network.segment_motion, bf16 and the command line end to end.

Tolerances.  Labels, count, dropped, area, box, centroid and peak are exact.  dx, dy are 64-bit fixed point at scale 2^S
(include/maskflow_b200.h): within 2^-(S+1) + 2^-50 (1 + |mean|) of the oracle's exact mean, NaN in the same places.
"""
import ctypes
import importlib.util
import os

import numpy as np
import pytest
import scipy.ndimage as ndi
import torch

from maskflownet_b200 import MaskflowError, _lib, network, ops
from maskflownet_b200.video import MotionFrame, VideoFlowPredictor, VideoMotionSegmenter
from oracle import motionseg_ref as R
from oracle import stabilize_ref as SR

from launchcheck.emu import build
from launchcheck.inputs import _deterministic
from launchcheck.motion_segment import _check, _mismatch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
EIGHT = np.ones((3, 3), int)


# ---------------------------------------------------------------------------------------------------------------
# inputs
# ---------------------------------------------------------------------------------------------------------------
def _spiral(H, W):
    m = np.zeros((H, W), bool)
    y0, x0, y1, x1 = 0, 0, H - 1, W - 1
    while y0 <= y1 and x0 <= x1:
        m[y0, x0:x1 + 1] = True
        m[y0:y1 + 1, x1] = True
        if y1 > y0 + 1:
            m[y1, x0:x1 + 1] = True
        if x1 > x0 + 1:
            m[y0 + 2:y1 + 1, x0] = True
        y0, x0, y1, x1 = y0 + 2, x0 + 2, y1 - 2, x1 - 2
        if y0 <= y1 and x0 - 1 <= x1:
            m[y0, x0 - 1] = True            # the step inwards that keeps the spiral one component
    return m


def _comb(H, W):
    m = np.zeros((H, W), bool)
    m[H - 1] = True
    m[:, ::2] = True
    return m


def _staircase(H, W):
    """Diagonal lines, connected only through corners; a second staircase of the other direction."""
    y, x = np.mgrid[0:H, 0:W]
    return ((x - y) % 7 == 0) | ((x + y) % 11 == 0)


def _checker(H, W):
    y, x = np.mgrid[0:H, 0:W]
    return (x + y) % 2 == 0


def _mask_inputs(mask, rng, hi_frac=0.2):
    """Residuals that put exactly `mask` above tau_lo = 1 (values in [1, 3), a share at least tau_hi = 2), the rest below
    (or NaN / occluded)."""
    N, H, W = mask.shape
    res = np.where(mask, rng.uniform(1.0, 2.0, mask.shape), rng.uniform(0.0, 0.99, mask.shape)).astype(np.float32)
    res[mask & (rng.random(mask.shape) < hi_frac)] += np.float32(1.0)
    return res


def _side_a(rng, N, H, W):
    flow = rng.normal(0, 4, (N, H, W, 2)).astype(np.float32)
    A = np.stack([_rot(rng) for _ in range(N)])
    return flow, A


def _rot(rng):
    c, s = np.cos(np.radians(rng.uniform(-2, 2))) * rng.uniform(0.98, 1.02), np.sin(np.radians(rng.uniform(-2, 2)))
    return np.array([[c, -s, rng.uniform(-5, 5)], [s, c, rng.uniform(-5, 5)]])


def _case(name, rng, N, H, W):
    """(res_a, occ_a, res_b, occ_b, flow_a, affine_a) and keyword arguments of one named case; every sample differs."""
    kw = dict(tau_lo=1.0, tau_hi=2.0, min_area=4, max_objects=255)
    shapes = {"spiral": _spiral, "comb": _comb, "staircase": _staircase, "checker": _checker}
    if name in shapes:
        m = np.stack([np.roll(shapes[name](H, W), n, axis=1) for n in range(N)])
    elif name == "full":
        m = np.ones((N, H, W), bool)
    elif name == "empty":
        m = np.zeros((N, H, W), bool)
    else:
        m = rng.random((N, H, W)) < rng.uniform(0.1, 0.6, (N, 1, 1))
    res_a = _mask_inputs(m, rng)
    res_b = _mask_inputs(m, rng)
    occ_a = (rng.random((N, H, W)) < 0.05).astype(np.uint8)
    occ_b = (rng.random((N, H, W)) < 0.05).astype(np.uint8)
    flow, A = _side_a(rng, N, H, W)
    if name == "nan":
        res_a[rng.random((N, H, W)) < 0.2] = np.nan
        res_b[rng.random((N, H, W)) < 0.2] = np.inf
    if name == "ties":
        # s exactly at tau_lo or tau_hi, and components of exactly min_area
        res_a = np.where(rng.random((N, H, W)) < 0.5, np.float32(1.0), np.float32(0.5)).astype(np.float32)
        res_a[rng.random((N, H, W)) < 0.1] = np.float32(2.0)
        res_b = res_a.copy()
        occ_a[:] = 0
        occ_b[:] = 0
        areas = [R.label(res_a[n] >= 1.0)[0] for n in range(N)]
        sizes = np.bincount(areas[0].ravel())[1:]
        kw["min_area"] = int(np.median(sizes)) if len(sizes) else 1
    if name == "many":
        kw.update(min_area=1, tau_hi=1.0, max_objects=7)
    if name == "a_null":
        res_a = occ_a = flow = A = None
    if name == "b_null":
        res_b = occ_b = None
    if name == "thresholds":
        kw.update(tau_lo=1.5, tau_hi=2.5, min_area=1, max_objects=100)
    return (res_a, occ_a, res_b, occ_b, flow, A), kw


CASES = ["random", "spiral", "comb", "staircase", "checker", "full", "empty", "nan", "ties", "many", "a_null", "b_null",
         "thresholds"]
HOST_SHAPES = [(2, 37, 53), (1, 1, 1), (1, 1, 70), (1, 70, 1), (2, 64, 96)]


def _oracle(inputs, kw, control=None):
    return R.segment(*inputs, control=control, **kw)


# ---------------------------------------------------------------------------------------------------------------
# the synthetic scene: a known affine camera, 0.3 px flow noise, NaN holes, a square moving 6 px and a disc moving 3 px
# relative to the camera
# ---------------------------------------------------------------------------------------------------------------
def _camera(H, W, pan=(4.0, -2.5), deg=0.5, zoom=1.01):
    c, s = zoom * np.cos(np.radians(deg)), zoom * np.sin(np.radians(deg))
    L = np.array([[c, -s], [s, c]])
    ctr = np.array([(W - 1) / 2, (H - 1) / 2])
    t = ctr - L @ ctr + np.array(pan)
    return np.concatenate([L, t[:, None]], 1)


def _inverse(A):
    L = np.linalg.inv(A[:, :2])
    return np.concatenate([L, -(L @ A[:, 2])[:, None]], 1)


def _objects(H, W, sx, sy):
    """The square and the disc of a frame, shifted by (sx, sy) px."""
    y, x = np.mgrid[0:H, 0:W].astype(np.float64)
    x, y = x - sx, y - sy
    a = 0.2 * min(H, W)
    square = (np.abs(x - 0.3 * W) <= a / 2) & (np.abs(y - 0.35 * H) <= a / 2)
    disc = (x - 0.7 * W) ** 2 + (y - 0.6 * H) ** 2 <= (0.12 * min(H, W)) ** 2
    return square, disc


V_SQUARE, V_DISC = np.array([4.8, -3.6]), np.array([0.0, 3.0])      # 6 px and 3 px


def scene(rng, H, W, camera=None):
    """Flows of frame t in both directions (flow_fw to frame t+1 and flow_bw to frame t-1), true occlusion masks (the
    background a moving object covers in the other frame) and the true object masks.  Returns (flows (2,H,W,2) float32
    forward then backward, occ (2,H,W) uint8, square, disc)."""
    A = _camera(H, W) if camera is None else camera
    Ab = _inverse(A)
    y, x = np.mgrid[0:H, 0:W].astype(np.float64)
    square, disc = _objects(H, W, 0, 0)
    flows, occ = np.empty((2, H, W, 2), np.float32), np.zeros((2, H, W), np.uint8)
    for k, (M, sign) in enumerate(((A, 1.0), (Ab, -1.0))):
        f = np.stack([M[0, 0] * x + M[0, 1] * y + M[0, 2] - x, M[1, 0] * x + M[1, 1] * y + M[1, 2] - y], -1)
        f[square] += sign * V_SQUARE
        f[disc] += sign * V_DISC
        f += rng.normal(0, 0.3, f.shape)
        f[rng.random((H, W)) < 0.01] = np.nan
        flows[k] = f
        cs, _ = _objects(H, W, *(sign * V_SQUARE))
        _, cd = _objects(H, W, *(sign * V_DISC))
        occ[k] = ((cs | cd) & ~(square | disc)).astype(np.uint8)
    return flows, occ, square, disc


def _scene_inputs(flows, occ, affine, residual):
    """ops.segment_motion's arguments for the scene's frame: side a the forward direction, side b the backward one."""
    return (residual[:1], occ[:1], residual[1:], occ[1:], flows[:1], affine[:1])


def _iou(a, b):
    return float((a & b).sum()) / float((a | b).sum())


def _scene_result(labels, count, square, disc):
    """(IoU of the square, IoU of the disc) when exactly two objects were found."""
    assert count == 2, count
    found = [labels == k for k in (1, 2)]
    # the square comes first in raster order (it lies higher in the frame)
    return _iou(found[0], square), _iou(found[1], disc)


SCENE_IOU = 0.99       # measured: at least 0.9988 over three seeds at the defaults


# ---------------------------------------------------------------------------------------------------------------
# the host build
# ---------------------------------------------------------------------------------------------------------------
def _ptr(a):
    return None if a is None else np.ascontiguousarray(a).ctypes.data_as(ctypes.c_void_p)


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    L = build(tmp_path_factory, "motionseg_emu")
    v, i = ctypes.c_void_p, ctypes.c_int
    L.emu_motion_segment.argtypes = [v] * 10 + [i] * 3 + [ctypes.c_float] * 2 + [i, i, ctypes.c_ulonglong]
    L.emu_union_find.argtypes = [v, v, i, i, i, ctypes.c_ulonglong]
    L.emu_workspace_bytes.argtypes = [i, i, i]
    L.emu_workspace_bytes.restype = ctypes.c_longlong
    L.emu_scale_bits.argtypes = [i, i]
    return L


def _host_segment(L, seed=0):
    def seg(res_a, occ_a, res_b, occ_b, flow_a, affine_a, tau_lo=1.0, tau_hi=2.0, min_area=64, max_objects=255):
        ref = res_a if res_a is not None else res_b
        N, H, W = ref.shape
        keep = [None if a is None else np.ascontiguousarray(a) for a in (res_a, occ_a, res_b, occ_b, flow_a, affine_a)]
        labels = np.zeros((N, H, W), np.uint8)
        objects = np.zeros((N, max_objects, 10))
        count, dropped = np.zeros(N, np.int32), np.zeros(N, np.int32)
        L.emu_motion_segment(*(_ptr(a) for a in keep), _ptr(labels), _ptr(objects), _ptr(count), _ptr(dropped), N, H, W,
                             tau_lo, tau_hi, min_area, max_objects, seed)
        return labels, objects, count, dropped
    return seg


def _gpu_segment():
    def seg(res_a, occ_a, res_b, occ_b, flow_a, affine_a, **kw):
        dev = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a)).cuda()   # noqa: E731
        out = ops.segment_motion(dev(res_a), dev(occ_a), dev(res_b), dev(occ_b), dev(flow_a), dev(affine_a), **kw)
        return tuple(t.cpu().numpy() for t in out)
    return seg


def _against_oracle(seg, N, H, W, seed):
    rng = np.random.default_rng(seed)
    for name in CASES:
        inputs, kw = _case(name, rng, N, H, W)
        _check(seg(*inputs, **kw), _oracle(inputs, kw), H, W, f"{name} {N}x{H}x{W}")


def _controls_fail(seg, N=2, H=48, W=64):
    """Each control of the oracle disagrees with the kernels on an input it concerns."""
    rng = np.random.default_rng(5)
    inputs, kw = _case("staircase", rng, N, H, W)
    assert _mismatch(seg(*inputs, **kw), _oracle(inputs, kw, "four_connected"), H, W) is not None
    inputs, kw = _case("random", rng, N, H, W)
    assert _mismatch(seg(*inputs, **kw), _oracle(inputs, kw, "max_score"), H, W) is not None


# ---------------------------------------------------------------------------------------------------------------
# CPU: the oracle's labelling
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("density", [0.1, 0.2, 0.3, 0.35, 0.4, 0.41, 0.45, 0.5, 0.6])
def test_oracle_labels_equal_scipy(density):
    """8-connected labels numbered in raster order of the first pixel, as scipy.ndimage.label numbers them; 0.41 is close
    to the site-percolation threshold of the 8-neighbour lattice (about 0.407), where components are largest."""
    rng = np.random.default_rng(int(density * 100))
    for H, W in ((1, 1), (1, 73), (73, 1), (37, 53), (256, 384)):
        m = rng.random((H, W)) < density
        got, n = R.label(m)
        want, nw = ndi.label(m, EIGHT)
        assert n == nw and np.array_equal(got, want), (H, W)
    for f in (_spiral, _comb, _staircase, _checker):
        m = f(61, 83)
        got, n = R.label(m)
        want, nw = ndi.label(m, EIGHT)
        assert n == nw and np.array_equal(got, want), f.__name__


def test_shapes_are_what_they_claim():
    assert ndi.label(_spiral(61, 83), EIGHT)[1] == 1 and ndi.label(_spiral(61, 83))[1] == 1
    assert ndi.label(_comb(40, 41), EIGHT)[1] == 1
    assert ndi.label(_checker(40, 41), EIGHT)[1] == 1 and ndi.label(_checker(40, 41))[1] == int(_checker(40, 41).sum())
    st = _staircase(61, 83)
    assert ndi.label(st)[1] > 5 * ndi.label(st, EIGHT)[1]      # 4-connectivity would split the corners


# ---------------------------------------------------------------------------------------------------------------
# CPU: the kernel source on the host
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N,H,W", HOST_SHAPES, ids=[f"{n}x{h}x{w}" for n, h, w in HOST_SHAPES])
def test_kernel_source_matches_oracle_on_host(emu, N, H, W):
    _against_oracle(_host_segment(emu), N, H, W, seed=H * 7 + W)


def test_union_order_does_not_matter_on_host(emu):
    """Shuffled orders of the unions, compression and statistics give the same result; every root is its component's
    first pixel (the find steps assert parent[i] < i on the host)."""
    rng = np.random.default_rng(3)
    N, H, W = 2, 53, 67
    for name in ("random", "spiral", "staircase", "checker", "nan"):
        inputs, kw = _case(name, rng, N, H, W)
        ref = _oracle(inputs, kw)
        for seed in (1, 2, 0xdeadbeef):
            _check(_host_segment(emu, seed)(*inputs, **kw), ref, H, W, f"{name}, order {seed}")
    m = np.stack([_spiral(H, W), rng.random((H, W)) < 0.41]).astype(np.uint8)
    for seed in (0, 7):
        roots = np.zeros((2, H, W), np.int32)
        emu.emu_union_find(_ptr(m), _ptr(roots), 2, H, W, seed)
        for n in range(2):
            flat = R.label(m[n])[0].ravel()
            idx = np.flatnonzero(flat)
            _, fi = np.unique(flat[idx], return_index=True)
            want = np.concatenate([[-1], idx[fi]])[flat]       # each pixel's component's first pixel
            assert np.array_equal(roots[n].ravel(), want)


def test_synthetic_scene_on_host(emu):
    rng = np.random.default_rng(11)
    H, W = 120, 160
    flows, occ, square, disc = scene(rng, H, W)
    affine, ok, residual = SR.fit(flows)
    assert ok.all()
    inputs = _scene_inputs(flows, occ, affine, residual)
    got = _host_segment(emu)(*inputs, min_area=ops.SEG_MIN_AREA)
    _check(got, R.segment(*inputs, min_area=ops.SEG_MIN_AREA), H, W, "scene")


def test_controls_fail_the_oracle_comparison_on_host(emu):
    _controls_fail(_host_segment(emu))


def test_workspace_formula(emu):
    L = _lib.lib()
    for N, H, W in ((1, 1, 1), (8, 436, 1024), (8, 1080, 1920), (3, 37, 53)):
        nb = L.mfn_motion_segment_workspace_bytes(N, H, W)
        assert nb == emu.emu_workspace_bytes(N, H, W)
        assert nb >= N * (4 * H * W + 12 * ((H + 1) // 2) * ((W + 1) // 2) + 255 * 64)
        assert nb <= N * (4 * H * W + 12 * ((H + 1) // 2) * ((W + 1) // 2) + 255 * 64 + 4 * H * W // 2048 + 64) + 6 * 256
    assert L.mfn_motion_segment_workspace_bytes(0, 3, 5) == 0
    assert emu.emu_scale_bits(1080, 1920) == R.scale_bits(1080, 1920) == 46 - 21


# ---------------------------------------------------------------------------------------------------------------
# CPU: the synthetic scene through the oracle
# ---------------------------------------------------------------------------------------------------------------
def test_synthetic_scene_through_the_oracle():
    """Both objects are found, nothing else, and the labels cover them; the camera-relative displacement of each object is
    its true motion within the noise."""
    rng = np.random.default_rng(2)
    H, W = 240, 320
    flows, occ, square, disc = scene(rng, H, W)
    affine, ok, residual = SR.fit(flows)
    labels, objects, count, dropped = R.segment(*_scene_inputs(flows, occ, affine, residual))
    iou = _scene_result(labels[0], count[0], square, disc)
    print(f"scene IoU: square {iou[0]:.4f}, disc {iou[1]:.4f}")
    assert min(iou) >= SCENE_IOU and dropped[0] == 0
    assert np.abs(objects[0, 0, 8:] - V_SQUARE).max() <= 0.1 and np.abs(objects[0, 1, 8:] - V_DISC).max() <= 0.1
    # side a alone also marks the background the square uncovers (the pixels its backward flow finds occluded)
    la, _, ca, _ = R.segment(residual[:1], occ[:1], None, None, flows[:1], affine[:1])
    assert ca[0] == 2 and _iou(la[0] == 1, square) < iou[0] - 0.005


# ---------------------------------------------------------------------------------------------------------------
# CPU: argument errors and the command line
# ---------------------------------------------------------------------------------------------------------------
def test_c_argument_errors_need_no_gpu():
    L = _lib.lib()
    buf = (ctypes.c_double * 4096)()
    p = ctypes.cast(buf, ctypes.c_void_p)
    odd = ctypes.c_void_p(p.value + 2)
    f = L.mfn_motion_segment

    def call(*, ptrs=None, nb=1 << 20, N=1, H=2, W=2, lo=1.0, hi=2.0, area=1, mo=255):
        ptrs = ptrs or [p] * 11
        return f(*ptrs, nb, N, H, W, lo, hi, area, mo, None)

    for k in (6, 7, 8, 9, 10):
        ptrs = [p] * 11
        ptrs[k] = None
        assert call(ptrs=ptrs) == -1 and b"null pointer" in L.mfn_last_error(), k
    for k in (0, 1, 4, 5):                         # an incomplete side a
        ptrs = [p] * 11
        ptrs[k] = None
        assert call(ptrs=ptrs) == -1 and b"go together" in L.mfn_last_error(), k
    for k in (2, 3):
        ptrs = [p] * 11
        ptrs[k] = None
        assert call(ptrs=ptrs) == -1 and b"go together" in L.mfn_last_error(), k
    for N, H, W in ((0, 2, 2), (1, 0, 2), (1, 2, -1)):
        assert call(N=N, H=H, W=W) == -1 and b"extent" in L.mfn_last_error()
    for lo, hi in ((2.0, 1.0), (float("nan"), 1.0), (1.0, float("inf")), (-float("inf"), 1.0)):
        assert call(lo=lo, hi=hi) == -1 and b"tau" in L.mfn_last_error(), (lo, hi)
    assert call(area=0) == -1 and b"min_area" in L.mfn_last_error()
    for mo in (0, 256, -1):
        assert call(mo=mo) == -1 and b"max_objects" in L.mfn_last_error()
    for k in (0, 2, 4, 5, 7, 8, 9, 10):
        ptrs = [p] * 11
        ptrs[k] = odd
        assert call(ptrs=ptrs) == -1 and b"aligned" in L.mfn_last_error(), k
    need = L.mfn_motion_segment_workspace_bytes(1, 2, 2)
    assert call(nb=need - 1) == -1 and b"workspace" in L.mfn_last_error()
    assert call(H=1 << 16, W=1 << 15, nb=1 << 40) == -3 and b"overflow" in L.mfn_last_error()
    assert call(N=65536, nb=1 << 40) == -3 and b"overflow" in L.mfn_last_error()


def test_ops_network_and_video_argument_errors_need_no_gpu():
    r = torch.zeros(1, 4, 4)
    o = torch.zeros(1, 4, 4, dtype=torch.uint8)
    for kw, msg in ((dict(tau_lo=2.0, tau_hi=1.0), "tau"), (dict(tau_lo=float("nan")), "tau"),
                    (dict(tau_hi=float("inf")), "tau"), (dict(tau_lo="x"), "tau"), (dict(min_area=0), "min_area"),
                    (dict(min_area=2.5), "min_area"), (dict(max_objects=0), "max_objects"),
                    (dict(max_objects=256), "max_objects"), (dict(max_objects=True), "max_objects")):
        with pytest.raises(MaskflowError, match=msg):
            ops.segment_motion(res_b=r, occ_b=o, **kw)
        with pytest.raises(MaskflowError, match=msg):
            VideoMotionSegmenter(torch.nn.Identity(), **kw)
    with pytest.raises(MaskflowError, match="go together"):
        ops.segment_motion(res_a=r, occ_a=o)
    with pytest.raises(MaskflowError, match="go together"):
        ops.segment_motion(res_b=r)
    with pytest.raises(MaskflowError, match="CUDA"):
        ops.segment_motion(res_b=r, occ_b=o)
    with pytest.raises(MaskflowError, match="shape"):
        ops.segment_motion()
    with pytest.raises(MaskflowError, match="batch"):
        VideoMotionSegmenter(torch.nn.Identity(), batch=0)
    s = VideoMotionSegmenter(torch.nn.Identity(), batch=4)
    assert s.bidirectional and s._outputs() == ("labels", "objects", "count", "dropped")
    with pytest.raises(MaskflowError, match="clip"):
        network.segment_motion(torch.nn.Identity(), torch.zeros(3, 4, 4, 3))
    with pytest.raises(MaskflowError, match="min_area"):
        network.segment_motion(torch.nn.Identity(), torch.zeros(3, 4, 4, 3, dtype=torch.uint8), min_area=0)


def _cli():
    spec = importlib.util.spec_from_file_location("segment_video", os.path.join(ROOT, "tools", "segment_video.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_command_line_arguments():
    cli = _cli()
    a = cli.parse_args(["objects.npz", "--video_filepath", "in.mp4", "-c", "w.params"])
    assert (a.tau_lo, a.tau_hi, a.min_area, a.batch, a.resize, a.precision, a.network, a.overlay) == \
        (ops.SEG_TAU_LO, ops.SEG_TAU_HI, ops.SEG_MIN_AREA, 8, None, "fp32", "MaskFlownet", None)
    a = cli.parse_args(["o.npz", "--video_filepath", "i.avi", "-c", "w.pt", "-n", "MaskFlownet_S", "--tau-lo", "0.5",
                        "--tau-hi", "3", "--min-area", "10", "--batch", "3", "--resize", "448,1024", "--precision", "bf16",
                        "--overlay", "o.avi"])
    assert (a.tau_lo, a.tau_hi, a.min_area, a.batch, a.resize, a.precision, a.network, a.overlay) == \
        (0.5, 3.0, 10, 3, (448, 1024), "bf16", "MaskFlownet_S", "o.avi")
    for bad in (["o.npz", "-c", "w"],
                ["o.npz", "--video_filepath", "i.mp4"],
                ["o.npz", "--video_filepath", "i.mp4", "-c", "w", "--tau-lo", "3", "--tau-hi", "2"],
                ["o.npz", "--video_filepath", "i.mp4", "-c", "w", "--min-area", "0"],
                ["o.npz", "--video_filepath", "i.mp4", "-c", "w", "--batch", "0"],
                ["o.npz", "--video_filepath", "i.mp4", "-c", "w", "--resize", "448"]):
        with pytest.raises(SystemExit):
            cli.parse_args(bad)
    rows = [np.zeros((0, 10)), np.arange(20.0).reshape(2, 10), np.ones((1, 10))]
    z = cli.pack_frames([MotionFrame(np.zeros((2, 3), np.uint8), r, d) for r, d in zip(rows, (0, 1, 0))])
    assert z["count"].tolist() == [0, 2, 1] and z["offset"].tolist() == [0, 0, 2] and z["dropped"].tolist() == [0, 1, 0]
    assert z["objects"].shape == (3, 10) and z["labels"].shape == (3, 2, 3) and list(z["columns"]) == list(R.COLUMNS)


# ---------------------------------------------------------------------------------------------------------------
# GPU: the kernels
# ---------------------------------------------------------------------------------------------------------------
GPU_SHAPES = [(8, 436, 1024), (8, 1080, 1920), (3, 37, 53), (1, 1, 257), (1, 257, 1), (1, 1, 1)]


@pytest.mark.gpu
@pytest.mark.parametrize("N,H,W", GPU_SHAPES, ids=[f"{n}x{h}x{w}" for n, h, w in GPU_SHAPES])
def test_kernels_match_oracle(N, H, W):
    _against_oracle(_gpu_segment(), N, H, W, seed=H + W)


def _scene_batch(rng, N, H, W):
    """N scenes of different cameras and noise, each frame's fit and residuals from ops.affine_motion."""
    flows, occ, masks = [], [], []
    for n in range(N):
        f, o, sq, di = scene(rng, H, W, _camera(H, W, pan=rng.uniform(-6, 6, 2), deg=rng.uniform(-1, 1),
                                                 zoom=rng.uniform(0.98, 1.02)))
        flows.append(f)
        occ.append(o)
        masks.append((sq, di))
    flows, occ = np.stack(flows), np.stack(occ)       # (N, 2, ...)
    fl = torch.from_numpy(np.concatenate([flows[:, 0], flows[:, 1]])).cuda()
    affine, ok, res = ops.affine_motion(fl, want_residual=True)
    assert bool(ok.all())
    res, affine = res.cpu().numpy(), affine.cpu().numpy()
    inputs = (res[:N], occ[:, 0].copy(), res[N:], occ[:, 1].copy(), flows[:, 0].copy(), affine[:N])
    return inputs, masks


@pytest.mark.gpu
@pytest.mark.parametrize("H,W", [(436, 1024), (1080, 1920)])
def test_synthetic_scene_on_gpu(H, W):
    rng = np.random.default_rng(H)
    inputs, masks = _scene_batch(rng, 8, H, W)
    got = _gpu_segment()(*inputs)
    _check(got, R.segment(*inputs), H, W, f"scene {H}x{W}")
    for n, (sq, di) in enumerate(masks):
        iou = _scene_result(got[0][n], got[2][n], sq, di)
        assert min(iou) >= SCENE_IOU, (n, iou)
    print(f"{H}x{W}: worst IoU {min(min(_scene_result(got[0][n], got[2][n], *masks[n])) for n in range(8)):.4f}")


@pytest.mark.gpu
def test_controls_fail_on_gpu():
    _controls_fail(_gpu_segment())


@pytest.mark.gpu
def test_reproducible_and_graph_replay():
    rng = np.random.default_rng(4)
    N, H, W = 8, 436, 1024
    inputs, kw = _case("random", rng, N, H, W)
    dev = [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in inputs]
    one = ops.segment_motion(*dev, **kw)
    two = ops.segment_motion(*dev, **kw)
    for a, b in zip(one, two):
        assert torch.equal(a.nan_to_num(), b.nan_to_num()) and torch.equal(a.isnan(), b.isnan())
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ops.segment_motion(*dev, **kw)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        cap = ops.segment_motion(*dev, **kw)
    for v in cap:
        v.zero_()
    n0 = _lib.launch_count()
    g.replay()
    torch.cuda.synchronize()
    assert _lib.launch_count() == n0               # a replay goes through no entry point
    for a, b in zip(cap, one):
        assert torch.equal(a.nan_to_num(), b.nan_to_num()) and torch.equal(a.isnan(), b.isnan())
    n0 = _lib.launch_count()
    ops.segment_motion(*dev, **kw)
    assert _lib.launch_count() - n0 == 11


@pytest.mark.gpu
def test_ops_argument_errors():
    r = torch.zeros(2, 8, 8, device="cuda")
    o = torch.zeros(2, 8, 8, dtype=torch.uint8, device="cuda")
    f = torch.zeros(2, 8, 8, 2, device="cuda")
    A = torch.zeros(2, 2, 3, dtype=torch.float64, device="cuda")
    for args in ((r.double(), o, f, A), (r, o.float(), f, A), (r, o, f[..., :1].contiguous(), A), (r, o, f, A.float()),
                 (r, o[:1], f, A), (r, o, f, A[:1]), (r.transpose(1, 2), o, f, A), (r[0], o, f, A)):
        with pytest.raises(MaskflowError, match="segment_motion"):
            ops.segment_motion(*args[:2], None, None, *args[2:])
    with pytest.raises(MaskflowError, match="forward-only"):
        ops.segment_motion(res_b=r.clone().requires_grad_(), occ_b=o)
    lab, obj, cnt, drp = ops.segment_motion(shape=(2, 5, 7), max_objects=3)
    assert lab.shape == (2, 5, 7) and not lab.any() and obj.shape == (2, 3, 10) and not obj.any()
    assert not cnt.any() and not drp.any()


# ---------------------------------------------------------------------------------------------------------------
# GPU: the network and the video segmenter
# ---------------------------------------------------------------------------------------------------------------
def _model(cls):
    torch.manual_seed(7)
    return cls().cuda().eval()


def _video(n, H, W, seed):
    """A textured background panning and a block moving across it."""
    g = np.random.default_rng(seed)
    bg = g.integers(0, 256, (H + 64, W + 64, 3)).astype(np.float64)
    bg = (bg + np.roll(bg, 1, 0) + np.roll(bg, 1, 1) + np.roll(bg, (1, 1), (0, 1))) / 4
    out = []
    for t in range(n):
        f = bg[2 * t % 32:2 * t % 32 + H, t % 32:t % 32 + W].copy()
        y0, x0 = H // 3, (W // 6 + 5 * t) % (W - H // 4)
        f[y0:y0 + H // 4, x0:x0 + H // 4] = g.integers(0, 256, 3)
        out.append(np.clip(np.rint(f), 0, 255).astype(np.uint8))
    return np.stack(out)


def _stream_equals_eager(seg, model, clip, what):
    got = list(seg.run(iter(clip)))
    assert len(got) == len(clip), (what, len(got))
    labels, objects, count, dropped = (t.cpu().numpy() for t in network.segment_motion(
        model, torch.from_numpy(clip).cuda(), batch=seg.batch, resize=seg.resize, **seg.seg_args))
    for t, fr in enumerate(got):
        assert isinstance(fr, MotionFrame) and fr.labels.shape == clip.shape[1:3] and fr.labels.dtype == np.uint8
        assert np.array_equal(fr.labels, labels[t]), (what, t)
        assert fr.objects.shape == (count[t], 10) and fr.dropped == dropped[t], (what, t)
        want = objects[t, :count[t]]
        assert np.array_equal(np.isnan(fr.objects), np.isnan(want)), (what, t)
        assert np.array_equal(np.nan_to_num(fr.objects), np.nan_to_num(want)), (what, t)
    last = objects[-1, :count[-1]]
    assert np.isnan(last[:, 8:]).all()             # the last frame has no side a
    return sum(int(c) for c in count)


@pytest.mark.gpu
@pytest.mark.parametrize("cls", [network.MaskFlownetS, network.MaskFlownet], ids=lambda c: c.__name__)
def test_video_segmenter_equals_eager_chain(cls):
    """Batch 4: 9 frames (two full batches), 11 frames (a partial last batch), run twice on the same segmenter, then 2
    and 1 frames."""
    model = _model(cls)
    H, W, resize = 100, 150, (128, 192)
    seg = VideoMotionSegmenter(model, batch=4, resize=resize, tau_lo=0.5, tau_hi=1.0, min_area=16)
    found = 0
    with _deterministic():
        for n, what in ((9, "9 frames"), (11, "11 frames"), (11, "11 frames again"), (2, "2 frames"), (1, "1 frame")):
            found += _stream_equals_eager(seg, model, _video(n, H, W, seed=n), what)
    print(f"{cls.__name__}: {found} objects over the clips")


@pytest.mark.gpu
def test_bf16_mode_and_video_predictor_unchanged():
    model = _model(network.MaskFlownetS)
    model.inference_precision = "bf16"
    clip = _video(7, 96, 128, seed=3)
    with _deterministic():
        _stream_equals_eager(VideoMotionSegmenter(model, batch=4, tau_lo=0.5, tau_hi=1.0, min_area=16), model, clip, "bf16")
    model.inference_precision = "fp32"
    got = list(VideoFlowPredictor(model, batch=4).run(iter(clip)))
    assert len(got) == len(clip) - 1 and got[0].shape == (96, 128, 3)


@pytest.mark.gpu
def test_segment_video_end_to_end(tmp_path):
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
    out, overlay = str(tmp_path / "objects.npz"), str(tmp_path / "overlay.avi")
    n = cli.segment_file(model, out, src, tau_lo=0.5, tau_hi=1.0, min_area=8, overlay=overlay, batch=4)
    assert n == len(frames)
    z = np.load(out)
    assert z["labels"].shape == (n, H, W) and z["count"].shape == (n,) and z["objects"].shape == (int(z["count"].sum()), 10)
    cap = cv2.VideoCapture(overlay)
    count = 0
    while True:
        ok, fr = cap.read()
        if not ok:
            break
        assert fr.shape == (H, W, 3)
        count += 1
    cap.release()
    assert count == n
