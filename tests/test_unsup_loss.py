"""Unsupervised fine-tuning: the census and smoothness loss kernels (csrc/unsup_loss.cu), their autograd Functions and
losses.unsupervised_loss, PipelineFlownet.train_batch_unsupervised and tools/finetune_unsupervised.py.

CPU: the kernel source compiled for the host (tests/host_emu/unsup_loss_emu.cpp) against the float64 oracle
(oracle/unsup_ref.py, its autograd for the gradients), the C entry points' argument errors, and the command line's
argument parsing and pair / crop sampling.  GPU: the same comparisons through ops at the training shapes, bit-identical
reruns, one network step against a float64 composition, free-flow recovery, an overfit run and the command line.

The bound (DESIGN.md section 2): |got - ref| <= u E / (1 - 64 u), u = 2^-24.  E is gamma_L S written out for a chain with
differences in it: every rounded intermediate x contributes (its number of fp32 roundings) * |x| * |d out / d x|, summed
over the chain in the kernel's order (a running error bound, first order).  The counts are derived from the source beside
each quantity in `census_bounds` / `smoothness_bounds`.  Where the kernels call powf / expf their documented error
(CUDA: 4 and 2 ulp) is added as kappa |value|.  Controls: one census offset dropped, the sign of the centre term of the
census backward flipped, the halo shifted by one pixel, the smoothness weighted by the other image's edges: each must
exceed the bound by at least 3x.
"""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from maskflownet_b200 import MaskflowError, _lib, losses, ops
from oracle import unsup_ref

from launchcheck.emu import build, ptr
from launchcheck.bounds import U
from launchcheck.unsup_loss import _d64, census_backward_control, census_bounds, ratio, smoothness_bounds

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, os.path.join(ROOT, "tools"))
CONTROL_RATIO = 3.0


# ---------------------------------------------------------------------------------------------------------------
# inputs
# ---------------------------------------------------------------------------------------------------------------
def make_images(rng, N, H, W):
    """img1, img2w (N,3,H,W) float32 in [0,1].  Even samples: smooth images (small grey differences, the steep part of
    the census transform) with img2w a slightly perturbed img1; odd samples: independent noise."""
    yy, xx = np.mgrid[0:H, 0:W]
    img1 = np.empty((N, 3, H, W))
    img2 = np.empty((N, 3, H, W))
    for n in range(N):
        if n % 2 == 0:
            base = np.stack([0.5 + 0.3 * np.sin(rng.uniform(0.05, 0.3) * xx + rng.uniform(0.05, 0.3) * yy + rng.uniform(0, 6))
                             for _ in range(3)])
            img1[n] = base + rng.normal(0, 0.004, base.shape)
            img2[n] = base + rng.normal(0, 0.004, base.shape) + 0.01 * rng.standard_normal()
        else:
            img1[n] = rng.random((3, H, W))
            img2[n] = np.where(rng.random((3, H, W)) < 0.5, img1[n] + rng.normal(0, 0.02, (3, H, W)), rng.random((3, H, W)))
    return np.clip(img1, 0, 1).astype(np.float32), np.clip(img2, 0, 1).astype(np.float32)


def make_occ(rng, N, H, W, kind):
    if kind == "none":
        return np.zeros((N, H, W), np.uint8)
    if kind == "all":
        return np.ones((N, H, W), np.uint8)
    return (rng.random((N, H, W)) < 0.3).astype(np.uint8)


def make_flow(rng, N, H, W):
    """A flow with smooth parts, kinks and exact zeros of the second difference (piecewise constant stretches)."""
    f = rng.normal(0, 2, (N, 2, H, W))
    f[:, :, :, : W // 3] = np.round(f[:, :, :, : W // 3])                       # integers: many exact zeros of d2x
    f[:, :, : H // 3] = np.repeat(f[:, :, :1], H // 3, axis=2) if H >= 3 else f[:, :, : H // 3]
    return f.astype(np.float32)


# ---------------------------------------------------------------------------------------------------------------
# checks against the float64 bounds (launchcheck/unsup_loss.py)
# ---------------------------------------------------------------------------------------------------------------
def check(got, ref, E, what):
    r = ratio(got, ref, E)
    assert r <= 1.0, f"{what}: |got - ref| is {r:.3g} x the bound"
    return r


def check_control(got, ref_control, E, what):
    r = ratio(got, ref_control, E)
    assert r >= CONTROL_RATIO, f"control {what}: only {r:.3g} x the bound"
    return r


def shift_x(img):
    """The image read one pixel to the right: what a halo staged one pixel off would give."""
    out = np.array(img, copy=True)
    out[..., :-1] = img[..., 1:]
    return out


# ---------------------------------------------------------------------------------------------------------------
# CPU: the kernel source on the host
# ---------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    L = build(tmp_path_factory, "unsup_loss_emu")
    L.emu_census_forward.argtypes = [ctypes.c_void_p] * 6 + [ctypes.c_int] * 3
    L.emu_census_distance.argtypes = [ctypes.c_void_p] * 3 + [ctypes.c_int] * 3
    L.emu_census_backward.argtypes = [ctypes.c_void_p] * 6 + [ctypes.c_int] * 3
    L.emu_smoothness_forward.argtypes = [ctypes.c_void_p] * 3 + [ctypes.c_int] * 3
    L.emu_smoothness_backward.argtypes = [ctypes.c_void_p] * 4 + [ctypes.c_int] * 3
    return L


class EmuKernels:
    def __init__(self, L):
        self.L = L

    def census(self, img1, img2w, occ):
        N, _, H, W = img1.shape
        coef = np.full((N, H, W), np.nan, np.float32)
        vsum, loss, d = np.zeros(N, np.float32), np.zeros(N, np.float32), np.zeros((N, H, W), np.float32)
        self.L.emu_census_forward(ptr(img1), ptr(img2w), ptr(occ), ptr(coef), ptr(vsum), ptr(loss), N, H, W)
        self.L.emu_census_distance(ptr(img1), ptr(img2w), ptr(d), N, H, W)
        return loss, vsum, coef, d

    def census_backward(self, img1, img2w, coef, vsum, g):
        gi = np.full(img2w.shape, np.nan, np.float32)
        N, _, H, W = img1.shape
        self.L.emu_census_backward(ptr(img1), ptr(img2w), ptr(coef), ptr(vsum), ptr(g), ptr(gi), N, H, W)
        return gi

    def smoothness(self, flow, img):
        N, _, H, W = flow.shape
        loss = np.full(N, np.nan, np.float32)
        self.L.emu_smoothness_forward(ptr(flow), ptr(img), ptr(loss), N, H, W)
        return loss

    def smoothness_backward(self, flow, img, g):
        N, _, H, W = flow.shape
        gf = np.full(flow.shape, np.nan, np.float32)
        self.L.emu_smoothness_backward(ptr(flow), ptr(img), ptr(g), ptr(gf), N, H, W)
        return gf


class GpuKernels:
    @staticmethod
    def _t(a):
        return torch.from_numpy(np.ascontiguousarray(a)).cuda()

    def census(self, img1, img2w, occ):
        loss, vsum, coef = ops._census_forward(self._t(img1), self._t(img2w), self._t(occ))
        return loss.cpu().numpy(), vsum.cpu().numpy(), coef.cpu().numpy(), None

    def census_backward(self, img1, img2w, coef, vsum, g):
        return ops._census_backward(self._t(img1), self._t(img2w), self._t(coef), self._t(vsum), self._t(g)).cpu().numpy()

    def smoothness(self, flow, img):
        return ops._smoothness_forward(self._t(flow), self._t(img)).cpu().numpy()

    def smoothness_backward(self, flow, img, g):
        return ops._smoothness_backward(self._t(flow), self._t(img), self._t(g)).cpu().numpy()


def run_census_checks(K, rng, N, H, W, occ_kind, controls=True):
    img1, img2w = make_images(rng, N, H, W)
    occ = make_occ(rng, N, H, W, occ_kind)
    g = rng.uniform(-2, 2, N).astype(np.float32)
    loss, vsum, coef, d = K.census(img1, img2w, occ)
    ref = census_bounds(img1, img2w, occ, g)
    assert np.array_equal(vsum, ref["vsum"].numpy().astype(np.float32))
    if d is not None:
        check(d, ref["d"], ref["E_d"], f"d {N}x{H}x{W}")
    check(coef, ref["coef"], ref["E_coef"], f"coef {N}x{H}x{W} occ={occ_kind}")
    check(loss, ref["loss"], ref["E_loss"], f"L_ph {N}x{H}x{W} occ={occ_kind}")
    gi = K.census_backward(img1, img2w, coef, vsum, g)
    check(gi, ref["grad"], ref["E_grad"], f"g_img2w {N}x{H}x{W} occ={occ_kind}")
    if H < 7 or W < 7:
        assert not loss.any() and not gi.any() and not coef.any()
    if not controls:
        return
    a, b, o = _d64(img1), _d64(img2w), torch.as_tensor(occ)
    ctl_d = unsup_ref.census_loss(a, b, o, offsets=unsup_ref.OFFSETS[:-1])[1]
    check_control(d if d is not None else coef, ctl_d if d is not None else
                  unsup_ref.census_loss(a, b, o, offsets=unsup_ref.OFFSETS[:-1])[3], ref["E_d" if d is not None else "E_coef"],
                  "dropped offset")
    check_control(gi, census_backward_control(img1, img2w, occ, g), ref["E_grad"], "centre sign flipped")
    sh = unsup_ref.census_loss(_d64(shift_x(img1)), _d64(shift_x(img2w)), o)
    check_control(coef, sh[3], ref["E_coef"], "halo shifted by one pixel")


def run_smoothness_checks(K, rng, N, H, W, controls=True):
    flow = make_flow(rng, N, H, W)
    img, other = make_images(rng, N, H, W)
    g = rng.uniform(-2, 2, N).astype(np.float32)
    loss = K.smoothness(flow, img)
    ref = smoothness_bounds(flow, img, g)
    check(loss, ref["loss"], ref["E_loss"], f"L_sm {N}x{H}x{W}")
    gf = K.smoothness_backward(flow, img, g)
    check(gf, ref["grad"], ref["E_grad"], f"g_flow {N}x{H}x{W}")
    if H < 3 and W < 3:
        assert not loss.any() and not gf.any()
    if controls:
        wrong = smoothness_bounds(flow, other, g)
        check_control(loss, wrong["loss"], ref["E_loss"], "smoothness weight from the other image")
        check_control(gf, wrong["grad"], ref["E_grad"], "smoothness weight from the other image (gradient)")


SMALL_SHAPES = [(1, 7, 7), (1, 6, 9), (2, 37, 53), (1, 1, 40), (1, 40, 1), (1, 8, 40)]


@pytest.mark.parametrize("occ_kind", ["none", "all", "random"])
def test_census_kernel_source_matches_oracle_on_host(emu, occ_kind):
    rng = np.random.default_rng(1)
    for N, H, W in SMALL_SHAPES:
        run_census_checks(EmuKernels(emu), rng, N, H, W, occ_kind,
                          controls=occ_kind != "all" and H >= 8 and W >= 8)


def test_smoothness_kernel_source_matches_oracle_on_host(emu):
    rng = np.random.default_rng(2)
    for N, H, W in SMALL_SHAPES + [(1, 2, 2), (1, 3, 1)]:
        run_smoothness_checks(EmuKernels(emu), rng, N, H, W, controls=H >= 8 and W >= 8)


def test_census_known_answers_on_host(emu):
    """Identical images: d = 0, rho = 1e-6^0.45, coef 0, gradient 0; everything occluded: loss 0, vsum 0."""
    K = EmuKernels(emu)
    rng = np.random.default_rng(3)
    img, _ = make_images(rng, 2, 12, 40)
    occ = np.zeros((2, 12, 40), np.uint8)
    loss, vsum, coef, d = K.census(img, img, occ)
    assert not d.any() and not coef.any() and np.all(vsum == 6 * 34)
    assert np.allclose(loss, 1e-6 ** 0.45, rtol=1e-5)
    loss, vsum, coef, _ = K.census(img, 1 - img, np.ones_like(occ))
    assert not loss.any() and not vsum.any() and not coef.any()


def test_argument_errors_need_no_gpu():
    L = _lib.lib()
    buf = (ctypes.c_float * 64)()
    p = ctypes.cast(buf, ctypes.c_void_p)
    odd = ctypes.c_void_p(p.value + 2)
    cf, cb = L.mfn_census_loss_forward, L.mfn_census_loss_backward
    sf, sb = L.mfn_smoothness_loss_forward, L.mfn_smoothness_loss_backward
    big = 1 << 20
    assert cf(None, p, p, p, p, p, p, big, 1, 8, 8, None) == -1 and b"null pointer" in L.mfn_last_error()
    assert cf(p, p, p, p, p, p, None, big, 1, 8, 8, None) == -1 and b"null pointer" in L.mfn_last_error()
    assert cb(p, p, p, p, p, None, 1, 8, 8, None) == -1 and b"null pointer" in L.mfn_last_error()
    assert sf(p, None, p, p, big, 1, 8, 8, None) == -1 and b"null pointer" in L.mfn_last_error()
    assert sb(p, p, None, p, 1, 8, 8, None) == -1 and b"null pointer" in L.mfn_last_error()
    for N, H, W in ((0, 8, 8), (1, 0, 8), (1, 8, -1)):
        assert cf(p, p, p, p, p, p, p, big, N, H, W, None) == -1 and b"extent" in L.mfn_last_error()
        assert cb(p, p, p, p, p, p, N, H, W, None) == -1 and b"extent" in L.mfn_last_error()
        assert sf(p, p, p, p, big, N, H, W, None) == -1 and b"extent" in L.mfn_last_error()
        assert sb(p, p, p, p, N, H, W, None) == -1 and b"extent" in L.mfn_last_error()
    assert cf(p, p, p, p, p, p, p, big, 65536, 8, 8, None) == -1 and b"overflow" in L.mfn_last_error()
    assert sb(p, p, p, p, 1, 1 << 15, 1 << 15, None) == -1 and b"overflow" in L.mfn_last_error()
    assert cf(odd, p, p, p, p, p, p, big, 1, 8, 8, None) == -1 and b"aligned" in L.mfn_last_error()
    assert cb(p, p, odd, p, p, p, 1, 8, 8, None) == -1 and b"aligned" in L.mfn_last_error()
    assert sf(p, p, p, odd, big, 1, 8, 8, None) == -1 and b"aligned" in L.mfn_last_error()
    assert sb(p, p, p, odd, 1, 8, 8, None) == -1 and b"aligned" in L.mfn_last_error()
    # workspace: 8 N ceil(H/8) ceil(W/32) (census), 8 N ceil(HW/256) (smoothness)
    need_c, need_s = ops.unsup_workspace_bytes("census", 2, 9, 33), ops.unsup_workspace_bytes("smoothness", 2, 9, 33)
    assert need_c == 8 * 2 * 2 * 2 and need_s == 8 * 2 * 2
    assert cf(p, p, p, p, p, p, p, need_c - 1, 2, 9, 33, None) == -1 and b"workspace" in L.mfn_last_error()
    assert sf(p, p, p, p, need_s - 1, 2, 9, 33, None) == -1 and b"workspace" in L.mfn_last_error()


# ---------------------------------------------------------------------------------------------------------------
# CPU: the command line
# ---------------------------------------------------------------------------------------------------------------
def _write_video(path, frames):
    import cv2
    h, w = frames[0].shape[:2]
    wr = cv2.VideoWriter(path, cv2.VideoWriter_fourcc(*"MJPG"), 10.0, (w, h))
    assert wr.isOpened()
    for f in frames:
        wr.write(f)
    wr.release()


def _video_frames(n, h, w, seed=0):
    rng = np.random.default_rng(seed)
    base = (rng.random((h + 8, w + 8 * n, 3)) * 255).astype(np.uint8)
    return [np.ascontiguousarray(base[4:4 + h, 3 * k:3 * k + w]) for k in range(n)]


def test_finetune_arguments_and_sampling(tmp_path):
    import finetune_unsupervised as ft
    vid = str(tmp_path / "v.avi")
    _write_video(vid, _video_frames(6, 72, 136))
    a = ft.parse_args(["--video_filepath", vid, "-c", "x.pt", "--crop", "64x128", "--batch", "3", "--steps", "2",
                       "-o", str(tmp_path / "out")])
    assert a.crop == (64, 128) and a.batch == 3 and a.steps == 2 and a.network == "MaskFlownet_S"
    for bad in (["--crop", "60x128"], ["--crop", "64"], ["--batch", "0"]):
        with pytest.raises(SystemExit):
            ft.parse_args(["--video_filepath", vid, "-c", "x.pt", "-o", "o"] + bad)
    with pytest.raises(SystemExit):
        ft.parse_args(["-c", "x.pt", "-o", "o"])                              # no input
    frames = ft.read_frames(video_filepath=vid)
    assert len(frames) == 6 and frames[0].shape == (72, 136, 3) and frames[0].dtype == np.uint8
    # BGR -> RGB: the first channel is what cv2 read as the last
    import cv2
    cap = cv2.VideoCapture(vid)
    ok, raw = cap.read()
    cap.release()
    assert ok and np.array_equal(frames[0], raw[..., ::-1])
    rng = np.random.default_rng(0)
    for _ in range(20):
        i1, i2, (idx, ys, xs) = ft.sample_batch(frames, 3, (64, 128), rng)
        assert i1.shape == (3, 3, 64, 128) and i1.dtype == np.uint8 and i2.shape == i1.shape
        for k in range(3):
            assert 0 <= idx[k] < len(frames) - 1 and 0 <= ys[k] <= 8 and 0 <= xs[k] <= 8
            want1 = frames[idx[k]][ys[k]:ys[k] + 64, xs[k]:xs[k] + 128].transpose(2, 0, 1)
            want2 = frames[idx[k] + 1][ys[k]:ys[k] + 64, xs[k]:xs[k] + 128].transpose(2, 0, 1)
            assert np.array_equal(i1[k], want1) and np.array_equal(i2[k], want2)      # consecutive frames, one crop
    frames_dir = tmp_path / "frames"
    frames_dir.mkdir()
    for k, f in enumerate(_video_frames(3, 64, 64)):
        cv2.imwrite(str(frames_dir / f"{k:03d}.png"), f)
    fr = ft.read_frames(frames_dir=str(frames_dir))
    assert len(fr) == 3 and fr[0].shape == (64, 64, 3)
    with pytest.raises(ValueError, match="crop"):
        ft.sample_batch(fr, 1, (128, 64), rng)
    with pytest.raises(ValueError, match="two frames"):
        ft.sample_batch(fr[:1], 1, (64, 64), rng)


# ---------------------------------------------------------------------------------------------------------------
# GPU: the kernels through ops
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("shape", [(8, 384, 512), (8, 320, 768)])
def test_census_and_smoothness_at_training_shapes(shape):
    rng = np.random.default_rng(10)
    run_census_checks(GpuKernels(), rng, *shape, "random")
    run_smoothness_checks(GpuKernels(), rng, *shape)


@pytest.mark.gpu
@pytest.mark.parametrize("occ_kind", ["none", "all", "random"])
def test_census_and_smoothness_small_shapes(occ_kind):
    rng = np.random.default_rng(11)
    for N, H, W in SMALL_SHAPES:
        run_census_checks(GpuKernels(), rng, N, H, W, occ_kind, controls=occ_kind != "all" and H >= 8 and W >= 8)
        run_smoothness_checks(GpuKernels(), rng, N, H, W, controls=H >= 8 and W >= 8)


@pytest.mark.gpu
def test_two_runs_are_bit_identical():
    rng = np.random.default_rng(12)
    img1, img2 = (torch.from_numpy(x).cuda() for x in make_images(rng, 8, 384, 512))
    flow = torch.from_numpy(make_flow(rng, 8, 384, 512)).cuda()
    occ = torch.from_numpy(make_occ(rng, 8, 384, 512, "random")).cuda()
    g = torch.from_numpy(rng.uniform(-2, 2, 8).astype(np.float32)).cuda()

    def run():
        loss, vsum, coef = ops._census_forward(img1, img2, occ)
        return (loss, vsum, coef, ops._census_backward(img1, img2, coef, vsum, g), ops._smoothness_forward(flow, img1),
                ops._smoothness_backward(flow, img1, g))
    first, second = run(), run()
    for x, y in zip(first, second):
        assert torch.equal(x, y)


@pytest.mark.gpu
def test_loss_functions_check_their_inputs():
    img = torch.rand(2, 3, 16, 16, device="cuda")
    occ = torch.zeros(2, 16, 16, dtype=torch.uint8, device="cuda")
    flow = torch.zeros(2, 2, 16, 16, device="cuda", requires_grad=True)
    with pytest.raises(MaskflowError, match="CUDA"):
        losses.census_loss(img.cpu(), img, occ)
    with pytest.raises(MaskflowError, match="contiguous"):
        losses.census_loss(img.transpose(2, 3), img, occ)
    with pytest.raises(MaskflowError, match="uint8"):
        losses.census_loss(img, img, occ.float())
    with pytest.raises(MaskflowError, match="shapes differ"):
        losses.census_loss(img, img[:1].contiguous(), occ)
    with pytest.raises(MaskflowError, match="data"):
        losses.census_loss(img.clone().requires_grad_(True), img, occ)
    with pytest.raises(MaskflowError, match="data"):
        losses.smoothness_loss(flow, img.clone().requires_grad_(True))
    with pytest.raises(MaskflowError, match="shapes differ"):
        losses.smoothness_loss(flow, img[:, :, :8].contiguous())
    with pytest.raises(MaskflowError, match=r"\(N,2,H,W\)"):
        losses.smoothness_loss(img, img)
    # autograd reaches img2_warped and the flow, and equals the direct backward calls
    w = img.flip(3).contiguous().requires_grad_(True)
    L = losses.census_loss(img, w, occ)
    L.sum().backward()
    loss, vsum, coef = ops._census_forward(img, w.detach(), occ)
    assert torch.equal(L.detach(), loss)
    assert torch.equal(w.grad, ops._census_backward(img, w.detach(), coef, vsum, torch.ones(2, device="cuda")))
    S = losses.smoothness_loss(flow, img)
    (2 * S).sum().backward()
    assert torch.equal(flow.grad, ops._smoothness_backward(flow.detach(), img, torch.full((2,), 2.0, device="cuda")))


# ---------------------------------------------------------------------------------------------------------------
# GPU: the loss on network flows, free-flow recovery, overfit, determinism, the command line
# ---------------------------------------------------------------------------------------------------------------
def _synthetic_batch(seeds, H, W, max_disp):
    from bf16_accuracy import synthetic_pair
    pairs = [synthetic_pair(s, H, W, max_disp) for s in seeds]
    return (torch.cat([p[0] for p in pairs]), torch.cat([p[1] for p in pairs]), torch.cat([p[2] for p in pairs]))


NETWORK_STEP_REL = 2.0 ** -10


def _gamma(L):
    return L * U / (1 - L * U)


def kernel_sample_positions(flow):
    """The sample positions (h, v) of ops.reconstruction2d on the fp32 flow (N, 2, H, W) (y, x) it reads, as the kernels
    compute them in fp32 (warp_fwd.cu), float64 values: the grid generator's g = fl(fl(fl(f + p) / s) - 1) with
    s = (W - 1) / 2 (exact), then the sampler's fl(fl(g + 1) * (W - 1)) / 2, one rounding per operation.  They lie within
    gamma_4 |f + p| + gamma_2 |f + p - s| px of f + p: the four relative roundings of the product chain, and the rounding
    of the grid g itself, relative to |g| = |f + p - s| / s, scaled back by s."""
    f = flow.detach().float().cpu()
    N, _, H, W = f.shape
    ys, xs = torch.arange(H, dtype=torch.float32).view(1, H, 1), torch.arange(W, dtype=torch.float32).view(1, 1, W)
    gy, gx = (f[:, 0] + ys) / ((H - 1) / 2) - 1, (f[:, 1] + xs) / ((W - 1) / 2) - 1
    return ((gy + 1) * (H - 1) / 2).double(), ((gx + 1) * (W - 1) / 2).double()


@pytest.mark.gpu
def test_network_step_gradient_matches_float64_composition():
    """The gradient of sum(unsupervised_loss) with respect to preds[-1] of a MaskFlownet-S training forward at batch 2N,
    against the oracle composition in float64: torch_ref.upsample, the zero-padded bilinear sample (the sampler) and
    oracle/unsup_ref.py on the same preds[-1] and the same occlusion masks (a data decision: both sides use the
    kernel's).  The random-init flows are scaled to at most 0.3 px, so that the two directions pass the consistency
    check (|w + w'|^2 <= 0.36 < beta) and the census sees the whole interior.  smooth_weight 0: Upsample(4) makes three
    of every four second differences zero in exact arithmetic, where the sign the smoothness gradient takes is decided
    by rounding; that term is held per element, sign allowance included, by the kernel tests above, and Upsample's
    backward by the existing operator tests.  Per element over the whole frame, |got - ref| <= 2^-10 S with
    S = Upsample(4)^T |dL/dF|: the gradient before the transposed Upsample's sum of up to 49 signed contributions cancels
    (the same kind of wiring bound DESIGN.md section 2 gives the cuDNN backward, with the census chain's steeper slope
    through the grey planes' rounding).
    The reference samples at the kernel's own fp32 positions (kernel_sample_positions, moving with F at slope 1), not at
    p + F: the grid generator's division and the sampler's de-normalisation round the position twice, up to ~1e-5 px
    where |g| is near 1, i.e. at the frame's edges.  Inside the frame that moves the sample by a neighbour difference
    times 1e-5; where a corner leaves the frame the zero padding makes the slope the whole pixel value, and the census
    (grey values x255 through D / sqrt(0.81 + D^2) and s^2 / (0.1 + s^2), second derivative up to ~20 at s = 0)
    turns that value change into a gradient change far above 2^-10 S (printed: up to ~29x in the last coarse row
    against the reference at p + F).  That the positions lie within their derived bound of p + F is asserted.
    Control: the two warps swapped (b warped by F_bw, a by F_fw) must exceed the bound by 3x."""
    from maskflownet_b200 import network
    from oracle import torch_ref
    torch.manual_seed(0)
    net = network.MaskFlownetS().cuda().train()
    a, b, _ = _synthetic_batch([1, 2], 256, 320, 4.0)
    a, b = a.cuda(), b.cuda()
    n = a.shape[0]
    x1, x2, _ = network.centralize(torch.cat([a, b]), torch.cat([b, a]))
    preds, _, _ = net(x1, x2)
    p = (preds[-1] * (0.3 / preds[-1].abs().max())).detach().clone().requires_grad_(True)
    flow = ops.upsample(p, 4)
    out = losses.unsupervised_loss(a, b, flow[:n], flow[n:], 0.0)
    out.loss.sum().backward()
    got = p.grad.double().cpu()
    with torch.no_grad():
        xy = lambda f: f.flip(1).permute(0, 2, 3, 1).contiguous()  # noqa: E731
        fl = flow.detach()
        occ = ops.flow_consistency(xy(fl[:n]), xy(fl[n:]))
    occ = tuple(o.cpu() for o in occ)
    a64, b64 = a.double().cpu(), b.double().cpu()
    H, W = a.shape[2:]
    h32, v32 = kernel_sample_positions(fl)
    ys = torch.arange(H, dtype=torch.float64).view(1, H, 1)
    xs = torch.arange(W, dtype=torch.float64).view(1, 1, W)
    f64 = fl.double().cpu()
    ey, ex = (h32 - (ys + f64[:, 0])).abs(), (v32 - (xs + f64[:, 1])).abs()
    sy, sx = (H - 1) / 2, (W - 1) / 2
    pos_ok = bool((ey <= _gamma(4) * (ys + f64[:, 0]).abs() + _gamma(2) * (ys + f64[:, 0] - sy).abs()).all()
                  and (ex <= _gamma(4) * (xs + f64[:, 1]).abs() + _gamma(2) * (xs + f64[:, 1] - sx).abs()).all())

    def ref_grad(swap_warps=False, fp32_positions=True):
        q = p.detach().double().cpu().requires_grad_(True)
        F = torch_ref.upsample(q, 4)
        F.retain_grad()
        fw, bw = (slice(n, None), slice(None, n)) if swap_warps else (slice(None, n), slice(n, None))

        def warp(x, rows):
            Fr = F[rows]
            if not fp32_positions:
                return torch_ref.reconstruction2d(x, Fr)
            return torch_ref.sample_tap(x, h32[rows] + (Fr[:, 0] - Fr[:, 0].detach()),
                                        v32[rows] + (Fr[:, 1] - Fr[:, 1].detach()), 1)
        b_w, a_w = warp(b64, fw), warp(a64, bw)
        L = unsup_ref.census_loss(torch.cat([a64, b64]), torch.cat([b_w, a_w]), torch.cat(occ).to(torch.uint8))[0]
        L.sum().backward()
        q2 = q.detach().clone().requires_grad_(True)
        (torch_ref.upsample(q2, 4) * F.grad.abs()).sum().backward()        # Upsample's weights are non-negative
        return q.grad, q2.grad
    ref, S = ref_grad()
    bound = NETWORK_STEP_REL * S
    ratio_map = (got - ref).abs() / bound
    worst = np.unravel_index(int(ratio_map.argmax()), tuple(ratio_map.shape))
    r = float(ratio_map.max())
    exact_map = (got - ref_grad(fp32_positions=False)[0]).abs() / bound
    worst_exact = np.unravel_index(int(exact_map.argmax()), tuple(exact_map.shape))
    r_ctl = float(((got - ref_grad(swap_warps=True)[0]).abs() / bound).max())
    print(f"network step: max|grad| {float(ref.abs().max()):.3e}, max S {float(S.max()):.3e}, max |got - ref| / bound "
          f"over the whole frame {r:.3g} at {worst}; with the reference sampling at p + F instead of the kernel's fp32 "
          f"positions {float(exact_map.max()):.3g} at {worst_exact}; positions off p + F by up to "
          f"{float(torch.maximum(ey, ex).max()):.3g} px; control {r_ctl:.3g}; occluded {float(out.occluded.mean()):.3f}")
    assert 0.0 < float(out.occluded.mean()) < 0.5
    assert pos_ok
    assert r <= 1.0 and r_ctl >= CONTROL_RATIO, (r, r_ctl)


_DET_SCRIPT = r"""
import sys, numpy as np, torch
from maskflownet_b200 import pipeline, augment
rng = np.random.default_rng(5)
img1 = rng.integers(0, 256, (2, 3, 128, 192), dtype=np.uint8)
img2 = np.roll(img1, 2, axis=3)
params = []
for run in range(2):
    torch.manual_seed(0)
    pipe = pipeline.PipelineFlownet(network_class="MaskFlownet_S", deterministic=True)
    col = augment.ColorAugmentation(contrast_range=(-0.4, 0.8), brightness_sigma=0.1, channel_range=(0.8, 1.4),
                                    batch_size=2, shape=(128, 192), noise_range=(0, 0.04), saturation=0.5, hue=0.5, seed=4)
    res = [pipe.train_batch_unsupervised(img1, img2, color_aug=col) for _ in range(3)]
    assert all(np.isfinite(r["loss"]) for r in res), res
    params.append([v.detach().clone() for v in pipe.network.state_dict().values()])
assert len(params[0]) > 0 and all(torch.equal(x, y) for x, y in zip(*params)), "parameters differ"
print("identical", res[-1])
"""


@pytest.mark.gpu
def test_unsupervised_step_is_bit_reproducible():
    env = dict(os.environ, CUBLAS_WORKSPACE_CONFIG=":4096:8", PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    flags = ["-s"] if sys.flags.no_user_site else []
    r = subprocess.run([sys.executable, *flags, "-c", _DET_SCRIPT], env=env, cwd=ROOT, capture_output=True, text=True)
    assert r.returncode == 0 and "identical" in r.stdout, r.stderr[-4000:]


@pytest.mark.gpu
def test_train_batch_unsupervised_checks_its_inputs():
    from maskflownet_b200 import pipeline
    pipe = pipeline.PipelineFlownet(network_class="MaskFlownet_S")
    u8 = np.zeros((1, 3, 64, 96), np.uint8)
    with pytest.raises(MaskflowError, match="multiples of 64"):
        pipe.train_batch_unsupervised(u8, u8)
    with pytest.raises(MaskflowError, match="uint8"):
        pipe.train_batch_unsupervised(np.zeros((1, 3, 64, 64), np.float32), np.zeros((1, 3, 64, 64), np.float32))


# free-flow recovery: both flows are leaves at 0, optimised with Adam on unsupervised_loss (no network)
# The same optimisation through the float64 oracle on the CPU (oracle/unsup_ref.py with torch_ref's sampler and its
# occlusion rule) sets the expectation.  Its EPE of F_fw against the known flow, every 50 steps:
#   1.2001 (0), 0.6258, 0.4185, 0.2979, 0.2217, 0.1722, 0.1383, 0.1157, 0.1007, 0.0906, 0.0836, 0.0783, 0.0750 (600)
# (smooth_weight 1.0 reached 0.2507 and 0.3 reached 0.5430 at 600 steps: README, "Unsupervised fine-tuning").
FREE_FLOW = dict(seed=0, H=128, W=192, max_disp=2.0, lr=0.05, steps=600, smooth_weight=3.0)
FREE_FLOW_CPU_FINAL_EPE = 0.0750


def free_flow_recovery(unsup, a, b, steps, lr, smooth_weight, make_leaf):
    """Returns the EPE curve of F_fw against the known flow (every 50 steps and the last)."""
    F_fw, F_bw = make_leaf(), make_leaf()
    opt = torch.optim.Adam([F_fw, F_bw], lr=lr)
    curve = []
    for s in range(steps + 1):
        if s % 50 == 0 or s == steps:
            curve.append((s, F_fw.detach().clone()))
        if s == steps:
            break
        opt.zero_grad()
        unsup(a, b, F_fw, F_bw, smooth_weight).sum().backward()
        opt.step()
    return curve


@pytest.mark.gpu
def test_free_flow_recovery():
    cfg = FREE_FLOW
    a, b, f = _synthetic_batch([cfg["seed"]], cfg["H"], cfg["W"], cfg["max_disp"])
    a, b = a.cuda(), b.cuda()
    curve = free_flow_recovery(lambda *args: losses.unsupervised_loss(*args).loss, a, b, cfg["steps"], cfg["lr"],
                               cfg["smooth_weight"], lambda: torch.zeros(1, 2, cfg["H"], cfg["W"], device="cuda",
                                                                         requires_grad=True))
    epe = [(s, float((F.cpu() - f).square().sum(1).sqrt().mean())) for s, F in curve]
    print("free-flow EPE curve (GPU):", [(s, round(e, 4)) for s, e in epe])
    e0, e1 = epe[0][1], epe[-1][1]
    assert e1 <= 0.25 * e0, epe
    assert abs(e1 - FREE_FLOW_CPU_FINAL_EPE) <= 0.1 * FREE_FLOW_CPU_FINAL_EPE, (e1, FREE_FLOW_CPU_FINAL_EPE)


@pytest.mark.gpu
def test_overfit_one_batch():
    """MaskFlownet-S from a seeded random initialisation, 200 steps on one batch of two synthetic pairs at 256x256.
    Adam at 1e-5: at 1e-4 the flows grow until every pixel fails the occlusion check, where the census term is empty
    and the loss falls to the smoothness alone while the EPE rises."""
    from maskflownet_b200 import pipeline
    torch.manual_seed(0)
    pipe = pipeline.PipelineFlownet(network_class="MaskFlownet_S", learning_rate=1e-5)
    a, b, f = _synthetic_batch([3, 4], 256, 256, 4.0)
    u1 = (a * 255).round().to(torch.uint8).numpy()
    u2 = (b * 255).round().to(torch.uint8).numpy()

    def epe():
        pipe.network.eval()
        with torch.no_grad():
            flow = network_predict(pipe, u1, u2)
        return float((flow.cpu() - f).square().sum(1).sqrt().mean())

    losses_, occl, epes = [], [], [epe()]
    for s in range(200):
        r = pipe.train_batch_unsupervised(u1, u2)
        losses_.append(r["loss"])
        occl.append(r["occluded"])
        if (s + 1) % 50 == 0:
            epes.append(epe())
    first, last = float(np.mean(losses_[:20])), float(np.mean(losses_[-20:]))
    print(f"overfit: loss every 10 steps {[round(x, 4) for x in losses_[::10]]}; mean first 20 {first:.4f}, "
          f"last 20 {last:.4f}; EPE every 50 steps {[round(e, 4) for e in epes]}; occluded every 10 steps "
          f"{[round(x, 3) for x in occl[::10]]}")
    assert last < first and epes[-1] < epes[0]


def network_predict(pipe, u1, u2):
    from maskflownet_b200 import network
    return network.predict_flow(pipe.network, torch.from_numpy(u1).cuda(), torch.from_numpy(u2).cuda())


@pytest.mark.gpu
def test_finetune_command_writes_a_loadable_checkpoint(tmp_path):
    import finetune_unsupervised as ft
    import predict_new_data
    from maskflownet_b200 import network
    torch.manual_seed(0)
    start = str(tmp_path / "start.pt")
    torch.save(network.MaskFlownetS().state_dict(), start)
    vid = str(tmp_path / "v.avi")
    _write_video(vid, _video_frames(5, 136, 200))
    out = str(tmp_path / "tuned")
    hist = ft.finetune(ft.parse_args(["--video_filepath", vid, "-c", start, "--crop", "128x192", "--batch", "2",
                                      "--steps", "3", "--color-aug", "-o", out]))
    assert len(hist) == 3 and all(np.isfinite(h["loss"]) for h in hist)
    before = torch.load(start)
    after = torch.load(out + ".pt")
    assert before.keys() == after.keys() and any(not torch.equal(before[k], after[k].cpu()) for k in before)
    model = predict_new_data.load_model("MaskFlownet_S", out + ".pt")
    frame = torch.from_numpy(_video_frames(2, 128, 192)[0]).permute(2, 0, 1)[None].contiguous().cuda()
    flow, _ = network.predict(model, frame, frame)
    assert flow.shape == (1, 128, 192, 2) and torch.isfinite(flow).all()
