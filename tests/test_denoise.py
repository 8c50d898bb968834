"""Video denoising: the kernels (csrc/denoise.cu, ops.denoise_frames, ops.estimate_noise), network.denoise_video,
video.VideoDenoiser and tools/denoise_video.py.

CPU: the kernel source compiled for the host (tests/host_emu/denoise_emu.cpp) against the float64 oracle
(oracle/denoise_ref.py) at several shapes and radii, in the ring form too; known answers; the gains on a synthetic scene
through the oracle, with a control that must lose; the noise estimate; argument errors and the command line.  GPU: the
same through the ops at the video sizes, reproducibility, batch independence, graph replay, a wrapping ring, and
VideoDenoiser bit for bit against network.denoise_video.

Tolerance.  The kernel walks the chains in float32 as the rule states, and so does the oracle; the oracle's samples,
colours, distances and weights are float64, the kernel's float32 (with fused multiply-adds on the GPU).  The value
before rounding therefore differs by about 1e-5 grey levels, which moves a result across a rounding tie only rarely:
outputs may differ by 1, and at least 99.9 % must be exact.  A chain decision (the frame edge or the round-trip test)
falls the other way where the round trip lies within float32 rounding of the threshold: the GPU contracts fb_sample's
lerps into fused multiply-adds, so its samples differ from the oracle's in the last bits.  The pixel then gains or loses
one neighbour, and its value may move by more than 1.  The test flows put many round trips near the threshold on
purpose; on the GPU at most FLIPPED = 1e-5 of the values may differ by more than 1 (at 8 x 436 x 1024, 99.999 % were exact),
on the host, which evaluates the kernel source without contraction, none may.  The noise estimate is an exact integer
sum and one float64 expression: bit-identical.
"""
import ctypes
import importlib.util
import os

import numpy as np
import pytest
import torch
from scipy.ndimage import binary_dilation, binary_erosion, gaussian_filter, map_coordinates

from maskflownet_b200 import MaskflowError, _lib, network, ops
from maskflownet_b200.video import VideoDenoiser, VideoFlowPredictor
from oracle import denoise_ref as R

from launchcheck.denoise import EXACT, FLIPPED, _case, _check  # noqa: F401
from launchcheck.emu import build, ptr
from launchcheck.inputs import _deterministic

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


# ---------------------------------------------------------------------------------------------------------------
# inputs: _case (launchcheck.denoise)
# ---------------------------------------------------------------------------------------------------------------
HOST_SHAPES = [(1, 1, 257), (1, 257, 1), (3, 37, 53), (2, 20, 40)]


# ---------------------------------------------------------------------------------------------------------------
# the host build and the two ways to run the kernels
# ---------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    L = build(tmp_path_factory, "denoise_emu")
    v, i, f = ctypes.c_void_p, ctypes.c_int, ctypes.c_float
    L.emu_denoise_frames.argtypes = [v] * 4 + [i] * 9 + [f] * 4
    L.emu_noise_sigma.argtypes = [v] * 3 + [i] * 3
    return L


def _host_ops(L):
    def denoise(frames, fw, bw, radius, sigma, h=ops.DENOISE_H, patch=ops.DENOISE_PATCH, t0=0, n=None, t_lo=0,
                t_hi=None, alpha=0.01, beta=0.5):
        S, H, W, _ = frames.shape
        t_hi = t_lo + S - 1 if t_hi is None else t_hi
        n = t_hi - t0 + 1 if n is None else n
        out = np.zeros((n, H, W, 3), np.uint8)
        frames, fw, bw = (np.ascontiguousarray(a) for a in (frames, fw, bw))
        L.emu_denoise_frames(ptr(frames), ptr(fw), ptr(bw), ptr(out), S, H, W, t0, n, t_lo, t_hi, radius, patch,
                             sigma, h, alpha, beta)
        return out

    def noise(frames):
        frames = np.ascontiguousarray(frames)
        F, H, W, _ = frames.shape
        s, S = np.zeros(F), np.zeros(F, np.int64)
        L.emu_noise_sigma(ptr(frames), ptr(s), ptr(S), F, H, W)
        return s, S
    return denoise, noise


def _gpu_ops():
    def denoise(frames, fw, bw, radius, sigma, h=ops.DENOISE_H, patch=ops.DENOISE_PATCH, t0=0, n=None, t_lo=0,
                t_hi=None, alpha=0.01, beta=0.5):
        d = [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in (frames, fw, bw)]
        return ops.denoise_frames(*d, radius, sigma, h, patch, alpha, beta, t0=t0, n=n, t_lo=t_lo,
                                  t_hi=t_hi).cpu().numpy()

    def noise(frames):
        return ops.estimate_noise(torch.from_numpy(np.ascontiguousarray(frames)).cuda()).cpu().numpy(), None
    return denoise, noise


def _against_oracle(denoise, N, H, W, radius, seed, patch=ops.DENOISE_PATCH, flipped=0.0):
    """N middle frames of an N + 2R clip (full windows) and the whole clip (windows clamped at both ends)."""
    rng = np.random.default_rng(seed)
    S = N + 2 * radius
    frames, fw, bw = _case(rng, S, H, W)
    got = denoise(frames, fw, bw, radius, 8.0, patch=patch, t0=radius, n=N)
    _check(got, R.denoise(frames, fw, bw, radius, 8.0, ops.DENOISE_H, patch, t0=radius, n=N), f"{N}x{H}x{W} R={radius}",
           flipped)
    if S <= 8 and H * W <= 40 * 60:
        got = denoise(frames, fw, bw, radius, 8.0, patch=patch)
        _check(got, R.denoise(frames, fw, bw, radius, 8.0, ops.DENOISE_H, patch), f"{N}x{H}x{W} R={radius} clip",
               flipped)


def _ring_equals_flat(denoise):
    """A 9-frame video held in a ring of 6 slots, frames 4..5 (t_lo = 2, t_hi = 8), equals the flat clip's."""
    rng = np.random.default_rng(11)
    T, H, W, S = 9, 24, 36, 6
    frames, fw, bw = _case(rng, T, H, W)
    flat = denoise(frames, fw, bw, 2, 8.0, t0=4, n=2, t_lo=2, t_hi=8)
    ring = [np.empty((S,) + a.shape[1:], a.dtype) for a in (frames, fw, bw)]
    for t in range(2, 8):                  # frames 2..7 in slots t % 6 (the window of 4..5 is 2..7)
        for dst, src in zip(ring, (frames, fw, bw)):
            dst[t % S] = src[t]
    got = denoise(*ring, 2, 8.0, t0=4, n=2, t_lo=2, t_hi=8)
    assert np.array_equal(got, flat)
    _check(got, R.denoise(*ring, 2, 8.0, ops.DENOISE_H, ops.DENOISE_PATCH, t0=4, n=2, t_lo=2, t_hi=8), "ring")


def _known_answers(denoise):
    rng = np.random.default_rng(3)
    T, H, W = 5, 23, 41
    frames = rng.integers(0, 256, (T, H, W, 3), dtype=np.uint8)
    zero = np.zeros((T, H, W, 2), np.float32)
    # R = 0 returns the input
    assert np.array_equal(denoise(frames, zero, zero, 0, 10.0), frames)
    # identical frames under zero flow
    same = np.repeat(frames[:1], T, 0)
    for patch in (0, 1, 3):
        assert np.array_equal(denoise(same, zero, zero, 2, 10.0, patch=patch), same)
    # every round trip fails: fw = bw = (1, 0)
    one = np.zeros((T, H, W, 2), np.float32)
    one[..., 0] = 1.0
    assert np.array_equal(denoise(frames, one, one, 3, 10.0), frames)
    # an integer pan of noise-free frames: frame t (y, x) = base[y + t, x + 2t]
    base = rng.integers(0, 256, (H + T, W + 2 * T, 3), dtype=np.uint8)
    pan = np.stack([base[t:t + H, 2 * t:2 * t + W] for t in range(T)])
    fw, bw = np.zeros((T, H, W, 2), np.float32), np.zeros((T, H, W, 2), np.float32)
    fw[..., 0], fw[..., 1], bw[..., 0], bw[..., 1] = -2, -1, 2, 1
    assert np.array_equal(denoise(pan, fw, bw, 2, 10.0), pan)


# ---------------------------------------------------------------------------------------------------------------
# the synthetic scene: a smooth textured background panning (1.3, 0.7) px per frame and a 40 px square moving
# (4.2, 2.1) px per frame against it, true flows, uint8 noise
# ---------------------------------------------------------------------------------------------------------------
SCENE_T, SCENE_H, SCENE_W = 7, 128, 192
BG, OBJ = np.array([-1.3, -0.7]), np.array([4.2, 2.1])


def scene(sigma, seed=0):
    """(clean (T,H,W,3) float64, noisy (T,H,W,3) uint8, square masks (T,H,W) bool)."""
    rng = np.random.default_rng(seed)
    H, W, T = SCENE_H, SCENE_W, SCENE_T
    canvas = gaussian_filter(rng.standard_normal((H + 80, W + 80, 3)), (2, 2, 0))
    canvas = (canvas - canvas.min()) / np.ptp(canvas) * 255
    obj = gaussian_filter(rng.standard_normal((40, 40, 3)), (1.5, 1.5, 0))
    obj = (obj - obj.min()) / np.ptp(obj) * 255
    yy, xx = np.mgrid[0:H, 0:W].astype(np.float64)
    clean, masks = [], []
    for t in range(T):
        img = np.stack([map_coordinates(canvas[..., c], [yy + 40 - BG[1] * t, xx + 40 - BG[0] * t], order=1)
                        for c in range(3)], -1)
        ox, oy = 60 + OBJ[0] * t, 40 + OBJ[1] * t
        m = (xx >= ox) & (xx < ox + 40) & (yy >= oy) & (yy < oy + 40)
        o = np.stack([map_coordinates(obj[..., c], [np.clip(yy - oy, 0, 39), np.clip(xx - ox, 0, 39)], order=1)
                      for c in range(3)], -1)
        img[m] = o[m]
        clean.append(img)
        masks.append(m)
    clean = np.stack(clean)
    noisy = np.clip(np.rint(clean + rng.normal(0, sigma, clean.shape)), 0, 255).astype(np.uint8)
    return clean, noisy, np.stack(masks)


def scene_flows(masks, missed=False):
    """True flows (fw of t -> t+1 and bw of t+1 -> t); with missed=True the square is given the background's motion."""
    T, H, W = masks.shape
    fw, bw = np.empty((T, H, W, 2), np.float32), np.empty((T, H, W, 2), np.float32)
    for t in range(T):
        fw[t] = np.where(masks[t][..., None] & (not missed), OBJ, BG)
        bw[t] = np.where(masks[min(t + 1, T - 1)][..., None] & (not missed), -OBJ, -BG)
    return fw, bw


def psnr(a, b, m=None):
    d = (np.asarray(a, np.float64) - b) ** 2
    return 10 * np.log10(255.0 ** 2 / (d[m] if m is not None else d).mean())


def scene_regions(mask):
    """The 8-px band around the square's boundary, and its interior eroded by 2 px."""
    return binary_dilation(mask, iterations=8) & ~binary_erosion(mask, iterations=8), binary_erosion(mask, iterations=2)


def scene_psnr(sigma, radius=ops.DENOISE_RADIUS, h=ops.DENOISE_H, patch=ops.DENOISE_PATCH, missed=False, seed=0):
    """PSNR of the middle frame through the oracle: (noisy, denoised) over the frame, the band and the interior."""
    clean, noisy, masks = scene(sigma, seed)
    fw, bw = scene_flows(masks, missed)
    t = SCENE_T // 2
    out = R.denoise(noisy, fw, bw, radius, sigma, h, patch, t0=t, n=1)[0]
    band, inner = scene_regions(masks[t])
    return {k: (psnr(noisy[t], clean[t], m), psnr(out, clean[t], m))
            for k, m in (("frame", None), ("band", band), ("object", inner))}


# ---------------------------------------------------------------------------------------------------------------
# CPU
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N,H,W", HOST_SHAPES, ids=lambda v: str(v))
def test_kernel_source_matches_oracle_on_host(emu, N, H, W):
    denoise, _ = _host_ops(emu)
    for radius in (0, 1, 2, 3):
        _against_oracle(denoise, N, H, W, radius, seed=N * 1000 + H + W + radius)


def test_patch_radii_and_ring_on_host(emu):
    denoise, _ = _host_ops(emu)
    for patch in (0, 2, 8):
        _against_oracle(denoise, 2, 21, 35, 2, seed=patch, patch=patch)
    _ring_equals_flat(denoise)


def test_known_answers_on_host(emu):
    _known_answers(_host_ops(emu)[0])


def test_noise_estimate_on_host(emu):
    _, noise = _host_ops(emu)
    rng = np.random.default_rng(5)
    for F, H, W in ((2, 37, 53), (1, 3, 3), (1, 3, 300), (1, 300, 3)):
        fr = rng.integers(0, 256, (F, H, W, 3), dtype=np.uint8)
        s, S = noise(fr)
        assert np.array_equal(S, R.noise_sums(fr)) and np.array_equal(s, R.noise_sigma(fr))
    flat = np.full((2, 20, 30, 3), 77, np.uint8)          # S = 0: the floor
    s, S = noise(flat)
    assert np.array_equal(S, [0, 0]) and np.array_equal(s, [ops.NOISE_FLOOR] * 2) and ops.NOISE_FLOOR == R.NOISE_FLOOR
    ramp = np.broadcast_to(np.arange(30, dtype=np.uint8)[None, None, :, None] * 3, (1, 20, 30, 3))
    assert np.array_equal(noise(ramp)[0], [ops.NOISE_FLOOR])   # a linear ramp has no second difference


def test_noise_estimate_within_3_percent_on_the_scene(emu):
    _, noise = _host_ops(emu)
    for sigma in (5, 10, 20):
        _, noisy, _ = scene(sigma, seed=1)
        s, _ = noise(noisy[:3])
        assert np.all(np.abs(s / sigma - 1) <= 0.03), (sigma, s)


def test_scene_gains_through_the_oracle():
    """True flows gain at least 6 dB; with the square's motion missed, the patch weights keep its interior within
    0.2 dB of the noisy input, and plain averaging along the flow (h -> inf), the control, loses more than 5 dB."""
    g = scene_psnr(10)
    assert g["frame"][1] - g["frame"][0] >= 6.0, g
    m = scene_psnr(10, missed=True)
    assert m["object"][1] >= m["object"][0] - 0.2, m
    c = scene_psnr(10, h=np.inf, missed=True)
    assert c["object"][1] < c["object"][0] - 5.0, c


def test_c_argument_errors_need_no_gpu():
    L = _lib.lib()
    buf = (ctypes.c_double * 256)()
    p = ctypes.cast(buf, ctypes.c_void_p)
    odd = ctypes.c_void_p(p.value + 4)
    f = L.mfn_denoise_frames

    def call(*, ptrs=None, S=5, H=2, W=2, t0=2, N=1, t_lo=0, t_hi=4, R=2, r=1, sigma=10.0, h=0.7, alpha=0.01,
             beta=0.5):
        return f(*(ptrs or [p] * 4), S, H, W, t0, N, t_lo, t_hi, R, r, sigma, h, alpha, beta, None)

    for k in range(4):
        ptrs = [p] * 4
        ptrs[k] = None
        assert call(ptrs=ptrs) == -1 and b"null pointer" in L.mfn_last_error(), k
    for kw in (dict(S=0), dict(H=0), dict(W=-1), dict(N=0)):
        assert call(**kw) == -1 and b"extent" in L.mfn_last_error(), kw
    for kw in (dict(R=-1), dict(r=-1)):
        assert call(**kw) == -1 and b"radius" in L.mfn_last_error(), kw
    for v in (0.0, -1.0, float("nan"), float("inf")):
        assert call(sigma=v) == -1 and b"sigma" in L.mfn_last_error(), v
        assert call(h=v) == -1 and b"h_factor" in L.mfn_last_error(), v
    for kw in (dict(alpha=-1.0), dict(beta=float("nan")), dict(alpha=float("inf"))):
        assert call(**kw) == -1 and b"alpha" in L.mfn_last_error(), kw
    for kw in (dict(t0=0, t_lo=1), dict(t0=4, N=2), dict(t_lo=-1, t0=0), dict(t0=-1)):
        assert call(**kw) == -1 and b"outside" in L.mfn_last_error(), kw
    assert call(S=4) == -1 and b"ring" in L.mfn_last_error()                     # frames 0..4 in 4 slots
    for k in (1, 2):
        ptrs = [p] * 4
        ptrs[k] = odd
        assert call(ptrs=ptrs) == -1 and b"aligned" in L.mfn_last_error(), k
    assert call(H=1 << 16, W=1 << 15) == -3 and b"overflow" in L.mfn_last_error()
    assert call(N=65536, t0=0, t_hi=70000, S=70000) == -3 and b"overflow" in L.mfn_last_error()
    assert call(r=9) == -2 and b"patch" in L.mfn_last_error()
    g = L.mfn_noise_sigma
    assert g(None, p, 1, 3, 3, None) == -1 and g(p, None, 1, 3, 3, None) == -1
    assert g(p, p, 0, 3, 3, None) == -1 and b"extent" in L.mfn_last_error()
    for H, W in ((2, 3), (3, 2), (1, 100)):
        assert g(p, p, 1, H, W, None) == -1 and b"interior" in L.mfn_last_error()
    assert g(p, odd, 1, 3, 3, None) == -1 and b"aligned" in L.mfn_last_error()
    assert g(p, p, 1, 1 << 16, 1 << 15, None) == -3 and g(p, p, 65536, 3, 3, None) == -3


def test_ops_network_and_video_argument_errors_need_no_gpu():
    fr = torch.zeros(5, 4, 4, 3, dtype=torch.uint8)
    fl = torch.zeros(5, 4, 4, 2)
    for kw, msg in ((dict(radius=-1), "radius"), (dict(radius=1.5), "radius"), (dict(sigma=0.0), "sigma"),
                    (dict(sigma=float("nan")), "sigma"), (dict(sigma=None), "sigma"), (dict(h=0.0), "h "),
                    (dict(h=float("inf")), "h "), (dict(patch=-1), "patch"), (dict(patch=9), "patch"),
                    (dict(alpha=-1.0), "alpha"), (dict(beta=float("inf")), "alpha")):
        args = dict(radius=2, sigma=10.0)
        args.update(kw)
        with pytest.raises(MaskflowError, match=msg):
            ops.denoise_frames(fr, fl, fl, **args)
    with pytest.raises(MaskflowError, match="CUDA"):
        ops.denoise_frames(fr, fl, fl, 2, 10.0)
    with pytest.raises(MaskflowError, match="CUDA"):
        ops.estimate_noise(fr)
    with pytest.raises(MaskflowError, match="uint8"):
        ops.estimate_noise(torch.zeros(4, 4))
    net = torch.nn.Identity()
    for kw, msg in ((dict(radius=-1), "radius"), (dict(sigma=0.0), "sigma"), (dict(h=-1.0), "h "),
                    (dict(patch=20), "patch"), (dict(batch=0), "batch")):
        with pytest.raises(MaskflowError, match=msg):
            VideoDenoiser(net, **kw)
        if "batch" not in kw:
            with pytest.raises(MaskflowError, match=msg):
                network.denoise_video(net, fr, **kw)
    d = VideoDenoiser(net, batch=4, radius=3)
    assert d._outputs() == () and d.bidirectional and d.ring_size == 2 * 3 + 2 * 4 + 1 and d.sigma is None
    assert d._segments(12, 17) == [(12, 15), (15, 17)] and d._segments(0, 3) == [(0, 3)]
    with pytest.raises(MaskflowError, match="clip"):
        network.denoise_video(net, torch.zeros(3, 4, 4, 3))
    with pytest.raises(MaskflowError, match="batch"):
        network.denoise_video(net, fr, batch=0)


def _cli():
    spec = importlib.util.spec_from_file_location("denoise_video", os.path.join(ROOT, "tools", "denoise_video.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_command_line_arguments():
    cli = _cli()
    a = cli.parse_args(["out.mp4", "--video_filepath", "in.mp4", "-c", "w.params"])
    assert (a.radius, a.sigma, a.h, a.patch, a.batch, a.resize, a.precision, a.network) == \
        (ops.DENOISE_RADIUS, None, ops.DENOISE_H, ops.DENOISE_PATCH, 8, None, "fp32", "MaskFlownet")
    a = cli.parse_args(["o.avi", "--video_filepath", "i.avi", "-c", "w.pt", "-n", "MaskFlownet_S", "--radius", "0",
                        "--sigma", "12.5", "--h", "1", "--patch", "2", "--batch", "3", "--resize", "448,1024",
                        "--precision", "bf16"])
    assert (a.radius, a.sigma, a.h, a.patch, a.batch, a.resize, a.precision, a.network) == \
        (0, 12.5, 1.0, 2, 3, (448, 1024), "bf16", "MaskFlownet_S")
    base = ["o.mp4", "--video_filepath", "i.mp4", "-c", "w"]
    for bad in (["o.mp4", "-c", "w"], ["o.mp4", "--video_filepath", "i.mp4"], base + ["--radius", "-1"],
                base + ["--sigma", "0"], base + ["--sigma", "inf"], base + ["--h", "0"], base + ["--patch", "9"],
                base + ["--patch", "-1"], base + ["--batch", "0"], base + ["--resize", "448"]):
        with pytest.raises(SystemExit):
            cli.parse_args(bad)


# ---------------------------------------------------------------------------------------------------------------
# GPU: the kernels
# ---------------------------------------------------------------------------------------------------------------
GPU_SHAPES = [(8, 436, 1024), (2, 1080, 1920), (3, 37, 53), (1, 1, 257), (1, 257, 1)]


@pytest.mark.gpu
@pytest.mark.parametrize("N,H,W", GPU_SHAPES, ids=lambda v: str(v))
def test_kernels_match_oracle(N, H, W):
    denoise, noise = _gpu_ops()
    big = H * W > 100000
    for radius in ((2,) if big else (0, 1, 2, 3)):
        _against_oracle(denoise, N, H, W, radius, seed=N + H + W + radius, flipped=FLIPPED)
    if big:                                  # R = 0, 1 and 3 on the middle frames of a shorter clip
        for radius in (0, 1, 3):
            _against_oracle(denoise, 1, H, W, radius, seed=radius, flipped=FLIPPED)
    if min(H, W) >= 3:
        fr = _case(np.random.default_rng(1), min(N + 1, 9), H, W)[0]
        assert np.array_equal(noise(fr)[0], R.noise_sigma(fr))


@pytest.mark.gpu
def test_known_answers_patch_radii_and_ring_on_gpu():
    denoise, noise = _gpu_ops()
    _known_answers(denoise)
    for patch in (0, 2, 8):
        _against_oracle(denoise, 2, 21, 35, 2, seed=patch, patch=patch, flipped=FLIPPED)
    _ring_equals_flat(denoise)
    assert np.array_equal(noise(np.full((2, 20, 30, 3), 77, np.uint8))[0], [ops.NOISE_FLOOR] * 2)
    for sigma in (5, 10, 20):
        _, noisy, _ = scene(sigma, seed=1)
        assert np.all(np.abs(noise(noisy[:3])[0] / sigma - 1) <= 0.03)


@pytest.mark.gpu
def test_reproducible_batch_independent_and_graph_replay():
    rng = np.random.default_rng(9)
    S, H, W = 10, 436, 1024
    frames, fw, bw = (torch.from_numpy(a).cuda() for a in _case(rng, S, H, W))
    a = ops.denoise_frames(frames, fw, bw, 3, 9.0)
    assert torch.equal(a, ops.denoise_frames(frames, fw, bw, 3, 9.0))
    for t0, n in ((0, 1), (4, 3), (9, 1)):                 # a frame's result does not depend on the others in the call
        assert torch.equal(ops.denoise_frames(frames, fw, bw, 3, 9.0, t0=t0, n=n), a[t0:t0 + n])
    out = torch.empty((4, H, W, 3), dtype=torch.uint8, device="cuda")
    sig = torch.empty((S,), dtype=torch.float64, device="cuda")
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        ops.denoise_frames(frames, fw, bw, 3, 9.0, t0=3, n=4, out=out)
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        ops.denoise_frames(frames, fw, bw, 3, 9.0, t0=3, n=4, out=out)
        sig.copy_(ops.estimate_noise(frames))
    out.zero_()
    sig.zero_()
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, a[3:7]) and torch.equal(sig, ops.estimate_noise(frames))


@pytest.mark.gpu
def test_ops_argument_errors():
    fr = torch.zeros(5, 4, 4, 3, dtype=torch.uint8, device="cuda")
    fl = torch.zeros(5, 4, 4, 2, device="cuda")
    with pytest.raises(MaskflowError, match="match"):
        ops.denoise_frames(fr, fl[:4], fl, 1, 10.0)
    with pytest.raises(MaskflowError, match="float32"):
        ops.denoise_frames(fr, fl.double(), fl, 1, 10.0)
    with pytest.raises(MaskflowError, match="outside"):
        ops.denoise_frames(fr, fl, fl, 1, 10.0, t0=3, n=3)
    with pytest.raises(MaskflowError, match="ring"):
        ops.denoise_frames(fr, fl, fl, 3, 10.0, t0=5, n=1, t_hi=10)
    with pytest.raises(MaskflowError, match="out"):
        ops.denoise_frames(fr, fl, fl, 1, 10.0, out=torch.empty(4, 4, 4, 3, dtype=torch.uint8, device="cuda"))
    with pytest.raises(MaskflowError, match="interior"):
        ops.estimate_noise(fr[:, :2].contiguous())
    assert ops.estimate_noise(fr[0]).shape == () and ops.median_noise(fr) == ops.NOISE_FLOOR


# ---------------------------------------------------------------------------------------------------------------
# GPU: the eager chain and the stream
# ---------------------------------------------------------------------------------------------------------------
def _model(cls):
    torch.manual_seed(7)
    return cls().cuda().eval()


def _video(n, H, W, seed):
    return _case(np.random.default_rng(seed), n, H, W, sigma=12.0)[0]


def _stream_equals_eager(den, model, clip, what):
    got = list(den.run(iter(clip)))
    assert len(got) == len(clip), (what, len(got))
    want, sigma = network.denoise_video(model, torch.from_numpy(clip).cuda(), batch=den.batch, resize=den.resize,
                                        radius=den.radius, sigma=den.sigma, h=den.h, patch=den.patch)
    assert sigma == den.sigma_used, (what, sigma, den.sigma_used)
    want = want.cpu().numpy()
    for t, fr in enumerate(got):
        assert fr.shape == clip.shape[1:] and fr.dtype == np.uint8
        assert np.array_equal(fr, want[t]), (what, t)
    return want


@pytest.mark.gpu
@pytest.mark.parametrize("cls", [network.MaskFlownetS, network.MaskFlownet], ids=lambda c: c.__name__)
def test_video_denoiser_equals_eager_chain(cls):
    """Batch 4: 11 frames (two full batches and a partial one), run twice on the same denoiser; then batch + 1, 2 and 1
    frames; radius 0, 1 and one longer than the video; a given sigma."""
    model = _model(cls)
    H, W, resize = 100, 150, (128, 192)
    with _deterministic():
        den = VideoDenoiser(model, batch=4, resize=resize, radius=2)
        clip = _video(11, H, W, seed=1)
        want = _stream_equals_eager(den, model, clip, "11 frames")
        assert (want != clip).mean() > 0.005     # the random network's flows pass the round trip in places
        _stream_equals_eager(den, model, clip, "11 frames again")
        for n in (5, 2, 1):
            _stream_equals_eager(den, model, _video(n, H, W, seed=n), f"{n} frames")
        one = _video(1, H, W, seed=3)
        assert np.array_equal(list(den.run(iter(one)))[0], one[0])
        for radius in (0, 1, 13):
            _stream_equals_eager(VideoDenoiser(model, batch=4, resize=resize, radius=radius), model, clip,
                                 f"radius {radius}")
        _stream_equals_eager(VideoDenoiser(model, batch=3, resize=resize, sigma=20.0, patch=2), model, clip,
                             "sigma 20, patch 2, batch 3")


@pytest.mark.gpu
def test_bf16_mode_and_video_predictor_unchanged():
    model = _model(network.MaskFlownetS)
    clip = _video(6, 96, 128, seed=3)
    with _deterministic():
        plain = list(VideoFlowPredictor(model, batch=4, bidirectional=True, want_flow=True).run(iter(clip)))
        assert len(plain) == len(clip) - 1
        P, dev_clip = len(clip) - 1, torch.from_numpy(clip).cuda()
        for k0 in range(0, P, 4):                 # the eager chain, batched and padded as the stream is
            x = dev_clip[[min(k0 + j, P) for j in range(5)]].permute(0, 3, 1, 2).contiguous()
            want = network.predict_bidirectional(model, x[:4], x[1:])
            for j in range(min(4, P - k0)):
                for got, ref in zip(plain[k0 + j][1:], want):
                    assert np.array_equal(got, ref[j].cpu().numpy()), (k0, j)
        model.inference_precision = "bf16"
        _stream_equals_eager(VideoDenoiser(model, batch=4, radius=2), model, clip, "bf16")
    model.inference_precision = "fp32"


@pytest.mark.gpu
def test_denoise_video_end_to_end(tmp_path):
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
    n, fps, sigma = cli.denoise_file(model, dst, src, radius=2, batch=4)
    assert n == len(frames) and fps == pytest.approx(12.0) and sigma >= ops.NOISE_FLOOR
    cap = cv2.VideoCapture(dst)
    count = 0
    while True:
        ok, fr = cap.read()
        if not ok:
            break
        assert fr.shape == (H, W, 3)
        count += 1
    cap.release()
    assert count == len(frames)
