"""Frame interpolation from bidirectional flow: the splatting kernels (csrc/interp.cu, ops.interpolate_frames),
network.interpolate_frames, VideoFlowPredictor(interpolate=T) and tools/interpolate_video.py.

CPU: the kernel source compiled for the host (tests/host_emu/interp_emu.cpp) against the float64 oracle
(oracle/interp_ref.py), known answers, order independence, four controls that must fail the comparison, the synthetic-scene
accuracy through the oracle, and argument errors.  GPU: the same through ops.interpolate_frames at the video sizes, the
network and video paths bit for bit against their eager chains, the command line, and the synthetic scene from the kernel.

Error bound (per output value, derived from interp.cu).  A contribution k of source weight w_k and bilinear factor b_k:
  * the fp32 factors (sampling.cuh, sampler_corners) are ax' = 1 - (q - floor q) and 1 - ax'.  Where |q| >= 1, q - floor q
    is a multiple of ulp(q) >= 2^-23, so both are exact; where |q| < 1 each may be off by 2^-25, so |ab' - ab| <= 2^-24
    + 2^-50 < DB = 2^-23 absolute, for contributions whose target has |qx| < 1 or |qy| < 1 (their w summed: wnear);
  * b' = fl(ax' ay'), w' = fl((1-t) ow), bw = fl(b' w') and the colour fl(bw I): four relative roundings of u = 2^-24;
  * the fixed-point conversion: 2^-(s_c+1) per colour and 2^-(s_w+1) per weight contribution (det.cuh), s_w = 61 - k,
    s_c = s_w - 8, k = bit length of 2HW.
The weight error enters the ratio r = C / W as (I_k - r) dW_k, |I_k - r| <= 255, so with n contributions and W the exact
weight sum:
    dW = DB wnear + 3 u W + n 2^-(s_w+1)
    |r' - r| <= (255 (DB wnear + 4 u W) + n 2^-s_c) / (W - dW)  +  2^-16 (the double and float roundings of the ratio).
A value within that of a rounding tie (k + 1/2), or a weight sum within dW of 2^-20, may round the other way: such values
are excluded and counted; every other value may differ by at most 1.  A hole's blend fmaf(t, I1, fl((1-t) I0)) is computed here exactly as the kernel rounds it, and
excluded where it lies on the other side of a tie from the exact blend.
"""
import ctypes
import importlib.util
import os

import numpy as np
import pytest
import torch

from maskflownet_b200 import MaskflowError, _lib, network, ops
from maskflownet_b200.video import VideoFlowPredictor
from oracle import interp_ref

from launchcheck.emu import build, ptr
from launchcheck.inputs import _deterministic
from launchcheck.interpolate import EXCLUDED_MAX, _check, _mismatch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
TIMES = (1e-3, 0.5, 0.999)


# ---------------------------------------------------------------------------------------------------------------
# inputs
# ---------------------------------------------------------------------------------------------------------------
def _case(rng, N, H, W, occ_kind="random"):
    """Images, flows and masks that exercise every branch: smooth motion, targets outside the frame, targets on the last
    row and column and on exact integers (at t = 1/2), NaN, +-inf and 1e30."""
    img0 = rng.integers(0, 256, (N, H, W, 3), dtype=np.uint8)
    img1 = rng.integers(0, 256, (N, H, W, 3), dtype=np.uint8)
    y, x = np.mgrid[0:H, 0:W]
    flows = []
    for sign in (1, -1):
        f = sign * rng.uniform(-0.2, 0.2, (N, 1, 1, 2)) * np.array([W, H]) + rng.normal(0, 0.7, (N, H, W, 2))
        m = rng.random((N, H, W)) < 0.1
        f[m] = rng.normal(0, 2 * max(H, W), (int(m.sum()), 2))                   # anywhere, often outside
        m = rng.random((N, H, W)) < 0.05
        f[..., 0] = np.where(m, 2.0 * ((W - 1) - x), f[..., 0])                   # x + u/2 = W - 1
        m = rng.random((N, H, W)) < 0.05
        f[..., 1] = np.where(m, 2.0 * ((H - 1) - y), f[..., 1])                   # y + v/2 = H - 1
        m = rng.random((N, H, W, 2)) < 0.05
        f[m] = 2.0 * rng.integers(-3, 4, int(m.sum()))                            # integer targets at t = 1/2
        m = rng.random((N, H, W, 2)) < 0.02
        f[m] = rng.choice([np.nan, np.inf, -np.inf, 1e30, -1e30], int(m.sum()))
        flows.append(f.astype(np.float32))
    if occ_kind == "zeros":
        occ = [np.zeros((N, H, W), np.uint8) for _ in range(2)]
    elif occ_kind == "ones":
        occ = [np.ones((N, H, W), np.uint8) for _ in range(2)]
    else:
        occ = [(rng.random((N, H, W)) < 0.3).astype(np.uint8) for _ in range(2)]
    return img0, img1, flows[0], flows[1], occ[0], occ[1]


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    L = build(tmp_path_factory, "interp_emu")
    L.emu_interpolate_frames.argtypes = [ctypes.c_void_p] * 7 + [ctypes.c_int] * 3 + [ctypes.c_void_p, ctypes.c_int,
                                                                                     ctypes.c_float] + [ctypes.c_void_p] * 2
    L.emu_interp_weight_shift.argtypes = [ctypes.c_int, ctypes.c_int]
    return L


def _emu_run(emu, img0, img1, ffw, fbw, ofw, obw, times, ow=0.01, order=None, want_acc=False):
    a = [np.ascontiguousarray(v) for v in (img0, img1, ffw, fbw, ofw, obw)]
    N, H, W, _ = a[0].shape
    ts = np.asarray(times, np.float32)
    out = np.full((N, len(ts), H, W, 3), 7, np.uint8)
    acc = np.zeros((N, H, W, 4), np.int64) if want_acc else None
    emu.emu_interpolate_frames(*(ptr(v) for v in a), ptr(out), N, H, W, ptr(ts), len(ts), ow,
                               None if order is None else ptr(order), None if acc is None else ptr(acc))
    return (out, acc) if want_acc else out


# ---------------------------------------------------------------------------------------------------------------
# known answers (any implementation: interp(img0, img1, flow_fw, flow_bw, occ_fw, occ_bw, times, occ_weight) -> numpy)
# ---------------------------------------------------------------------------------------------------------------
def _known_answers(interp):
    rng = np.random.default_rng(11)
    N, H, W = 2, 19, 27
    img = rng.integers(0, 256, (N, H, W, 3), dtype=np.uint8)
    z = np.zeros((N, H, W, 2), np.float32)
    occ = (rng.random((N, H, W)) < 0.5).astype(np.uint8)
    for ow in (0.01, 0.0, 1.0):                          # identical frames, zero flow: the frame itself
        got = interp(img, img, z, z, occ, occ[::-1].copy(), TIMES, ow)
        assert np.array_equal(got, np.broadcast_to(img[:, None], got.shape)), ow
    other = rng.integers(0, 256, (N, H, W, 3), dtype=np.uint8)
    zero = np.zeros((N, H, W), np.uint8)
    for t, d in ((0.5, (4, -2)), (0.25, (4, -8)), (0.75, (-4, 4))):   # integer translation with t d integral
        img1 = np.roll(img, (d[1], d[0]), axis=(1, 2))
        f = np.broadcast_to(np.array(d, np.float32), z.shape).copy()
        got = interp(img, img1, f, -f, zero, zero, (t,), 0.01)[:, 0]
        sx, sy = int(t * d[0]), int(t * d[1])
        want = np.roll(img, (sy, sx), axis=(1, 2))
        m = max(abs(d[0]), abs(d[1]))
        assert np.array_equal(got[:, m:H - m, m:W - m], want[:, m:H - m, m:W - m]), (t, d)
    blend_t = (0.25, 0.5, 0.75)                          # exact in float32: the kernel's blend rounds exactly
    tt = np.asarray(blend_t, np.float32).astype(np.float64)[None, :, None, None, None]
    blend = np.rint((1.0 - tt) * img[:, None] + tt * other[:, None]).astype(np.uint8)
    far = np.full((N, H, W, 2), 1e4, np.float32)         # every target outside the frame
    assert np.array_equal(interp(img, other, far, -far, zero, zero, blend_t, 0.01), blend)
    flow = rng.normal(0, 2, (N, H, W, 2)).astype(np.float32)
    ones = np.ones((N, H, W), np.uint8)                  # everything occluded at occ_weight 0
    assert np.array_equal(interp(img, other, flow, -flow, ones, ones, blend_t, 0.0), blend)
    ofw, obw = (rng.random((2, N, H, W)) < 0.3).astype(np.uint8)   # T times in one call = T single-time calls
    many = interp(img, other, flow, flow[::-1].copy(), ofw, obw, TIMES, 0.01)
    for k, t in enumerate(TIMES):
        assert np.array_equal(many[:, k], interp(img, other, flow, flow[::-1].copy(), ofw, obw, (t,), 0.01)[:, 0]), t


# ---------------------------------------------------------------------------------------------------------------
# the synthetic scene: true flows and the true middle frame (background moves (2,2) px, a 40 x 40 square (12,6) px)
# ---------------------------------------------------------------------------------------------------------------
SCENE_OW = (0.01, 0.001, 0.1, 1.0, 0.0)


def _scene():
    from scipy.ndimage import binary_dilation, gaussian_filter
    rng = np.random.default_rng(0)
    H, W = 128, 192

    def tex(h, w, s):
        t = np.stack([gaussian_filter(rng.standard_normal((h, w)), s) for _ in range(3)], -1)
        return np.rint((t - t.min()) / (t.max() - t.min()) * 255).astype(np.uint8)

    bg, fg = tex(H + 40, W + 40, 2.0), tex(40, 40, 1.0)
    dbg, dfg, fy0, fx0 = np.array([2, 2]), np.array([12, 6]), 40, 60

    def render(t):
        oy, ox = int(t * dbg[1]), int(t * dbg[0])
        im = bg[20 - oy:20 - oy + H, 20 - ox:20 - ox + W].copy()
        y, x = fy0 + int(t * dfg[1]), fx0 + int(t * dfg[0])
        im[y:y + 40, x:x + 40] = fg
        return im

    def flow(t, sign):
        f = np.zeros((H, W, 2), np.float32)
        f[:] = sign * dbg
        y, x = fy0 + int(t * dfg[1]), fx0 + int(t * dfg[0])
        f[y:y + 40, x:x + 40] = sign * dfg
        return f

    fgm = np.zeros((H, W), bool)
    fgm[fy0 + 3:fy0 + 43, fx0 + 6:fx0 + 46] = True
    band = binary_dilation(fgm, iterations=8) ^ ~binary_dilation(~fgm, iterations=8)
    f01, f10 = flow(0, 1), flow(1, -1)
    return render(0), render(1), render(0.5), f01, f10, _fb_occ(f01, f10), _fb_occ(f10, f01), band


def _fb_occ(f, o, alpha=0.01, beta=0.5):
    """The forward-backward check (ops.flow_consistency's rule) in float64, for one (H,W,2) flow against the other."""
    H, W, _ = f.shape
    y, x = np.mgrid[0:H, 0:W]
    qx, qy = x + f[..., 0].astype(np.float64), y + f[..., 1].astype(np.float64)
    inside = (qx >= 0) & (qx <= W - 1) & (qy >= 0) & (qy <= H - 1)
    qx, qy = np.clip(qx, 0, W - 1), np.clip(qy, 0, H - 1)
    x0, y0 = np.floor(qx).astype(int), np.floor(qy).astype(int)
    x1, y1 = np.minimum(x0 + 1, W - 1), np.minimum(y0 + 1, H - 1)
    wx, wy = (qx - x0)[..., None], (qy - y0)[..., None]
    g = o.astype(np.float64)
    b = (g[y0, x0] * (1 - wx) + g[y0, x1] * wx) * (1 - wy) + (g[y1, x0] * (1 - wx) + g[y1, x1] * wx) * wy
    d2 = ((f + b) ** 2).sum(-1)
    m2 = (f.astype(np.float64) ** 2).sum(-1) + (b ** 2).sum(-1)
    return (~(inside & (d2 <= alpha * m2 + beta))).astype(np.uint8)


def _psnr(a, b, m=None):
    d = (a.astype(np.float64) - b.astype(np.float64)) ** 2
    d = d[m] if m is not None else d
    return 10 * np.log10(255.0 ** 2 / d.mean())


def _scene_table(interp):
    """{occ_weight: (PSNR whole frame, PSNR band, hole share)} and the no-flow blend's (whole, band), at t = 1/2.
    interp(img0, img1, f01, f10, o0, o1, ow) -> ((H,W,3) uint8 frame, hole share or None)."""
    i0, i1, ih, f01, f10, o0, o1, band = _scene()
    rows = {}
    for ow in SCENE_OW:
        out, holes = interp(i0, i1, f01, f10, o0, o1, ow)
        rows[ow] = (_psnr(out, ih), _psnr(out, ih, band), holes)
    blend = np.rint(0.5 * i0.astype(np.float64) + 0.5 * i1).astype(np.uint8)
    rows["blend"] = (_psnr(blend, ih), _psnr(blend, ih, band), None)
    for k, (a, b, h) in rows.items():
        print(f"occ_weight {k!s:6}: whole {a:6.2f} dB, band {b:6.2f} dB" + (f", holes {100 * h:.3f} %" if h is not None
                                                                               else ""))
    return rows


def _oracle_scene(i0, i1, f01, f10, o0, o1, ow):
    r = interp_ref.interpolate(i0[None], i1[None], f01[None], f10[None], o0[None], o1[None], (0.5,), ow)
    return r["frames"][0, 0], float(r["hole"].mean())


def _check_scene_table(rows):
    assert rows[0.01][1] >= rows[1.0][1] + 6.0, rows          # beats plain average splatting in the band
    assert rows[0.01][0] >= rows["blend"][0] + 15.0, rows     # beats the no-flow blend overall


# ---------------------------------------------------------------------------------------------------------------
# CPU: the kernel source on the host
# ---------------------------------------------------------------------------------------------------------------
def test_kernel_source_matches_oracle_on_host(emu):
    rng = np.random.default_rng(0)
    excluded = total = 0
    for N, H, W in ((1, 1, 1), (1, 1, 29), (1, 23, 1), (2, 37, 53)):
        for occ_kind in ("zeros", "ones", "random"):
            for ow in (0.0, 0.01, 1.0):
                args = _case(rng, N, H, W, occ_kind)
                got = _emu_run(emu, *args, TIMES, ow)
                ref = interp_ref.interpolate(*args, TIMES, ow)
                e, n = _check(got, ref, args[0], args[1], TIMES, f"{N}x{H}x{W} {occ_kind} ow={ow}")
                excluded, total = excluded + e, total + n
    print(f"excluded {excluded} of {total} values")
    assert excluded <= EXCLUDED_MAX * total, (excluded, total)


def test_weight_scale_is_61_minus_fanin_bits(emu):
    for H, W in ((1, 1), (37, 53), (436, 1024), (2160, 3840)):
        assert emu.emu_interp_weight_shift(H, W) == 61 - int(2 * H * W).bit_length(), (H, W)


def test_known_answers_on_host(emu):
    _known_answers(lambda *a: _emu_run(emu, *a))


def test_order_independence_on_host(emu):
    rng = np.random.default_rng(3)
    N, H, W = 2, 21, 33
    args = _case(rng, N, H, W)
    threads = 2 * N * ((H * W + 255) // 256) * 256
    out0, acc0 = _emu_run(emu, *args, (0.3,), 0.01, want_acc=True)
    for seed in (1, 2):
        order = np.random.default_rng(seed).permutation(threads).astype(np.int64)
        out1, acc1 = _emu_run(emu, *args, (0.3,), 0.01, order=order, want_acc=True)
        assert np.array_equal(acc0, acc1) and np.array_equal(out0, out1), seed


@pytest.mark.parametrize("control", ["drop_corner", "swap_weights", "move_by_t", "other_mask"])
def test_controls_fail_the_oracle_comparison(emu, control):
    """Each control changes the rule in one place; the kernel must disagree with it on many values, far outside the
    exclusions, while it agrees with the rule itself."""
    rng = np.random.default_rng(5)
    N, H, W = 2, 37, 53
    args = _case(rng, N, H, W)
    got = _emu_run(emu, *args, (0.3,), 0.01)
    assert _mismatch(got, interp_ref.interpolate(*args, (0.3,), 0.01), args[0], args[1], (0.3,))[0] == 0
    ctl = interp_ref.interpolate(*args, (0.3,), 0.01, control=control)
    bad, excl, total, _ = _mismatch(got, ctl, args[0], args[1], (0.3,))
    print(f"control {control}: {bad} of {total} values differ")
    assert bad >= 0.05 * total, (control, bad, total)


def test_synthetic_scene_through_the_oracle():
    _check_scene_table(_scene_table(_oracle_scene))


# ---------------------------------------------------------------------------------------------------------------
# CPU: argument errors
# ---------------------------------------------------------------------------------------------------------------
def test_c_argument_errors_need_no_gpu():
    L = _lib.lib()
    buf = (ctypes.c_float * 256)()
    p = ctypes.cast(buf, ctypes.c_void_p)
    odd = ctypes.c_void_p(p.value + 4)
    ts = (ctypes.c_float * 2)(0.25, 0.5)
    tsp = ctypes.cast(ts, ctypes.c_void_p)
    f = L.mfn_interpolate_frames
    assert L.mfn_interpolate_frames_workspace_bytes(2, 3, 5) == 32 * 2 * 3 * 5
    assert L.mfn_interpolate_frames_workspace_bytes(0, 3, 5) == 0

    def call(*, ptrs=None, ws=p, nb=1024, N=1, H=2, W=2, times=tsp, T=2, ow=0.01):
        ptrs = ptrs or [p] * 7
        return f(*ptrs, ws, nb, N, H, W, times, T, ow, None)

    for k in range(7):
        ptrs = [p] * 7
        ptrs[k] = None
        assert call(ptrs=ptrs) == -1 and b"null pointer" in L.mfn_last_error(), k
    assert call(ws=None) == -1 and b"null pointer" in L.mfn_last_error()
    assert call(times=None) == -1 and b"null pointer" in L.mfn_last_error()
    for N, H, W in ((0, 2, 2), (1, 0, 2), (1, 2, -1)):
        assert call(N=N, H=H, W=W) == -1 and b"extent" in L.mfn_last_error()
    assert call(T=0) == -1 and b"T must" in L.mfn_last_error()
    for bad in (0.0, 1.0, -0.5, 1.5, float("nan"), float("inf")):
        tb = ctypes.cast((ctypes.c_float * 2)(0.5, bad), ctypes.c_void_p)
        assert call(times=tb) == -1 and b"outside (0,1)" in L.mfn_last_error(), bad
    for ow in (-0.01, 1.01, float("nan"), float("inf")):
        assert call(ow=ow) == -1 and b"occ_weight" in L.mfn_last_error(), ow
    for k in (2, 3):
        ptrs = [p] * 7
        ptrs[k] = odd
        assert call(ptrs=ptrs) == -1 and b"aligned" in L.mfn_last_error(), k
    assert call(ws=ctypes.c_void_p(p.value + 8)) == -1 and b"aligned" in L.mfn_last_error()
    assert call(nb=32 * 4 - 1) == -1 and b"workspace" in L.mfn_last_error()
    assert call(H=1 << 16, W=1 << 15) == -3 and b"overflow" in L.mfn_last_error()
    assert call(N=65536) == -3 and b"overflow" in L.mfn_last_error()


def test_ops_and_video_argument_errors_need_no_gpu():
    img = torch.zeros(1, 4, 4, 3, dtype=torch.uint8)
    flow = torch.zeros(1, 4, 4, 2)
    occ = torch.zeros(1, 4, 4, dtype=torch.uint8)
    for times in ((), (0.0,), (1.0,), (0.5, float("nan")), 1.5):
        with pytest.raises(MaskflowError, match="time"):
            ops.interpolate_frames(img, img, flow, flow, occ, occ, times)
    for ow in (-0.1, 1.5, float("nan")):
        with pytest.raises(MaskflowError, match="occ_weight"):
            ops.interpolate_frames(img, img, flow, flow, occ, occ, 0.5, ow)
    with pytest.raises(MaskflowError, match="CUDA"):
        ops.interpolate_frames(img, img, flow, flow, occ, occ, 0.5)
    net = torch.nn.Identity()
    for bad in (-1, 1.5, True, "2"):
        with pytest.raises(MaskflowError, match="interpolate"):
            VideoFlowPredictor(net, interpolate=bad)
    for ow in (-0.5, 2.0, float("nan")):
        with pytest.raises(MaskflowError, match="occ_weight"):
            VideoFlowPredictor(net, interpolate=1, occ_weight=ow)
    p = VideoFlowPredictor(net, interpolate=3)
    assert p.bidirectional and p._outputs() == ("frames",)
    p = VideoFlowPredictor(net, interpolate=1, want_flow=True)
    assert p._outputs() == ("frames", "flow", "flow_bw", "occ_fw", "occ_bw")
    assert VideoFlowPredictor(net)._outputs() == ("rgb",) and not VideoFlowPredictor(net).bidirectional


def _cli():
    spec = importlib.util.spec_from_file_location("interpolate_video", os.path.join(ROOT, "tools", "interpolate_video.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_command_line_arguments():
    cli = _cli()
    a = cli.parse_args(["out.mp4", "--video_filepath", "in.mp4", "-c", "w.params", "--factor", "4"])
    assert (a.factor, a.batch, a.resize, a.precision, a.fps, a.network) == (4, 8, None, "fp32", None, "MaskFlownet")
    a = cli.parse_args(["o.avi", "--video_filepath", "i.avi", "-c", "w.pt", "-n", "MaskFlownet_S", "--factor", "2",
                        "--batch", "3", "--resize", "448,1024", "--precision", "bf16", "--fps", "24"])
    assert (a.factor, a.batch, a.resize, a.precision, a.fps, a.network) == (2, 3, (448, 1024), "bf16", 24.0,
                                                                            "MaskFlownet_S")
    for bad in (["o.mp4", "--video_filepath", "i.mp4", "-c", "w", "--factor", "1"],
                ["o.mp4", "--video_filepath", "i.mp4", "-c", "w"],
                ["o.mp4", "-c", "w", "--factor", "2"],
                ["o.mp4", "--video_filepath", "i.mp4", "-c", "w", "--factor", "2", "--batch", "0"],
                ["o.mp4", "--video_filepath", "i.mp4", "-c", "w", "--factor", "2", "--resize", "448"],
                ["o.mp4", "--video_filepath", "i.mp4", "-c", "w", "--factor", "2", "--fps", "0"]):
        with pytest.raises(SystemExit):
            cli.parse_args(bad)


# ---------------------------------------------------------------------------------------------------------------
# GPU: the kernel
# ---------------------------------------------------------------------------------------------------------------
def _gpu_run(img0, img1, ffw, fbw, ofw, obw, times, ow=0.01):
    t = [torch.from_numpy(np.ascontiguousarray(v)).cuda() for v in (img0, img1, ffw, fbw, ofw, obw)]
    return ops.interpolate_frames(*t, times, ow).cpu().numpy()


GPU_SHAPES = [(3, 37, 53, 3), (8, 436, 1024, 1), (1, 1080, 1920, 7), (1, 2160, 3840, 1)]


@pytest.mark.gpu
@pytest.mark.parametrize("N,H,W,T", GPU_SHAPES, ids=[f"{n}x{h}x{w}-T{t}" for n, h, w, t in GPU_SHAPES])
def test_kernel_matches_oracle(N, H, W, T):
    rng = np.random.default_rng(H)
    args = _case(rng, N, H, W)
    times = [(k + 1) / (T + 1) for k in range(T)] if T > 1 else [0.37]
    got = _gpu_run(*args, times)
    e, n = _check(got, interp_ref.interpolate(*args, times, 0.01), args[0], args[1], times, f"{N}x{H}x{W}")
    print(f"{N}x{H}x{W} T={T}: excluded {e} of {n} values")
    assert e <= EXCLUDED_MAX * n, (e, n)


@pytest.mark.gpu
def test_known_answers_repeatability_and_single_pair():
    _known_answers(_gpu_run)
    args = _case(np.random.default_rng(8), 4, 64, 96)
    t = [torch.from_numpy(np.ascontiguousarray(v)).cuda() for v in args]
    a = ops.interpolate_frames(*t, TIMES)
    b = ops.interpolate_frames(*t, TIMES)
    assert torch.equal(a, b)
    one = ops.interpolate_frames(*(v[1] for v in t), TIMES)
    assert one.shape == (3, 64, 96, 3) and torch.equal(one, a[1])


@pytest.mark.gpu
def test_ops_argument_errors():
    img = torch.zeros(2, 8, 8, 3, dtype=torch.uint8, device="cuda")
    flow = torch.zeros(2, 8, 8, 2, device="cuda")
    occ = torch.zeros(2, 8, 8, dtype=torch.uint8, device="cuda")
    ok = [img, img, flow, flow, occ, occ]
    for k, bad in ((0, img.float()), (2, flow.double()), (4, occ.bool()), (2, flow.transpose(1, 2)),
                   (0, img[..., :2].contiguous()), (3, flow[:1]), (5, occ[:, :7].contiguous()), (1, img.cpu())):
        a = list(ok)
        a[k] = bad
        with pytest.raises(MaskflowError, match="interpolate_frames"):
            ops.interpolate_frames(*a, 0.5)
    with pytest.raises(MaskflowError, match="forward-only"):
        ops.interpolate_frames(img, img, flow.clone().requires_grad_(), flow, occ, occ, 0.5)


@pytest.mark.gpu
def test_synthetic_scene_from_the_kernel():
    def kernel(i0, i1, f01, f10, o0, o1, ow):
        return _gpu_run(i0[None], i1[None], f01[None], f10[None], o0[None], o1[None], (0.5,), ow)[0, 0], None

    i0, i1, ih, f01, f10, o0, o1, band = _scene()
    g0, g1 = ops.flow_consistency(torch.from_numpy(f01).cuda(), torch.from_numpy(f10).cuda())
    assert np.array_equal(g0.cpu().numpy(), o0) and np.array_equal(g1.cpu().numpy(), o1)
    ref, got = _scene_table(_oracle_scene), _scene_table(kernel)
    _check_scene_table(got)
    for k in ref:
        assert abs(ref[k][0] - got[k][0]) <= 0.01 and abs(ref[k][1] - got[k][1]) <= 0.01, (k, ref[k], got[k])


# ---------------------------------------------------------------------------------------------------------------
# GPU: the network and the video predictor
# ---------------------------------------------------------------------------------------------------------------
def _model(cls):
    torch.manual_seed(7)
    return cls().cuda().eval()


NET_CASES = [(network.MaskFlownetS, 1, 64, 64), (network.MaskFlownetS, 2, 448, 1024), (network.MaskFlownet, 1, 64, 64),
             (network.MaskFlownet, 2, 448, 1024)]


@pytest.mark.gpu
@pytest.mark.parametrize("cls,n,H,W", NET_CASES, ids=[f"{c.__name__}-{n}x{h}x{w}" for c, n, h, w in NET_CASES])
def test_network_interpolate_frames_equals_its_chain(cls, n, H, W):
    model = _model(cls)
    g = np.random.default_rng(H + n)
    a, b = (torch.from_numpy(g.integers(0, 256, (n, 3, H, W), dtype=np.uint8)).cuda() for _ in range(2))
    with _deterministic():
        got = network.interpolate_frames(model, a, b, (0.25, 0.5))
        fw, bw, ofw, obw = network.predict_bidirectional(model, a, b)
        want = ops.interpolate_frames(a.permute(0, 2, 3, 1).contiguous(), b.permute(0, 2, 3, 1).contiguous(), fw, bw, ofw,
                                      obw, (0.25, 0.5))
    assert got.shape == (n, 2, H, W, 3) and got.dtype == torch.uint8
    assert torch.equal(got, want)


def _frames(n, H, W, seed):
    return np.random.default_rng(seed).integers(0, 256, (n, H, W, 3), dtype=np.uint8)


VIDEO_CASES = [(network.MaskFlownetS, 1, True), (network.MaskFlownetS, 3, False), (network.MaskFlownet, 3, True)]


@pytest.mark.gpu
@pytest.mark.parametrize("cls,T,want_flow", VIDEO_CASES, ids=[f"{c.__name__}-T{t}-{w}" for c, t, w in VIDEO_CASES])
def test_video_predictor_interpolate_graph_equals_eager_chain(cls, T, want_flow):
    """7 frames at batch 4 (one full batch and one of 2 pairs), then a 3-frame video (shorter than one batch): every
    result equals, bit for bit, predict_bidirectional + ops.interpolate_frames run eagerly on the same 4-pair batch (the
    last one padded with the last frame)."""
    model = _model(cls)
    B, resize, H, W = 4, (128, 192), 100, 150
    times = [k / (T + 1) for k in range(1, T + 1)]
    with _deterministic():
        pred = VideoFlowPredictor(model, batch=B, resize=resize, want_flow=want_flow, interpolate=T)
        for frames in (_frames(7, H, W, seed=4), _frames(3, H, W, seed=5)):
            P = len(frames) - 1
            got = list(pred.run(iter(frames)))
            assert len(got) == P
            for k in range((P + B - 1) // B):
                idx = [min(B * k + j, P) for j in range(B + 1)]
                Fh = torch.from_numpy(frames[idx]).cuda()
                x = Fh.permute(0, 3, 1, 2).contiguous()
                fw, bw, ofw, obw = network.predict_bidirectional(model, x[:B], x[1:], resize)
                want = ops.interpolate_frames(Fh[:B], Fh[1:], fw, bw, ofw, obw, times)
                for j in range(min(B, P - B * k)):
                    r = got[B * k + j]
                    stack = r[0] if want_flow else r
                    assert stack.shape == (T, H, W, 3) and stack.dtype == np.uint8
                    assert np.array_equal(stack, want[j].cpu().numpy()), (len(frames), B * k + j)
                    if want_flow:
                        for g, e, nm in ((r[1], fw, "flow"), (r[2], bw, "flow_bw"), (r[3], ofw, "occ_fw"),
                                         (r[4], obw, "occ_bw")):
                            assert np.array_equal(g, e[j].cpu().numpy()), (len(frames), B * k + j, nm)


@pytest.mark.gpu
def test_interpolate_video_end_to_end(tmp_path):
    cv2 = pytest.importorskip("cv2")
    cli = _cli()
    model = _model(network.MaskFlownetS)
    H = W = 64
    frames = _frames(5, H, W, seed=6)
    src = str(tmp_path / "in.avi")
    wr = cv2.VideoWriter(src, cv2.VideoWriter_fourcc(*"MJPG"), 10.0, (W, H))
    for f in frames:
        wr.write(f)
    wr.release()
    for factor, fps, batch in ((3, None, 2), (2, 10.0, 8)):
        dst = str(tmp_path / f"out{factor}.avi")
        n, fps_out = cli.interpolate_file(model, dst, src, factor, batch=batch, fps=fps)
        assert n == (len(frames) - 1) * factor + 1 and fps_out == pytest.approx(fps or 10.0 * factor)
        cap = cv2.VideoCapture(dst)
        assert cap.get(cv2.CAP_PROP_FPS) == pytest.approx(fps_out)
        count = 0
        while True:
            ok, fr = cap.read()
            if not ok:
                break
            assert fr.shape == (H, W, 3)
            count += 1
        cap.release()
        assert count == n, (factor, count, n)
