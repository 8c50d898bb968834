"""Middlebury colour coding of flows (csrc/flowvis.cu, ops.flow_to_color), the streaming video predictor built on it
(maskflownet_b200/video.py) and the predict_new_data command line (tools/predict_new_data.py).

CPU: the kernel source compiled for the host (tests/host_emu/flowvis_emu.cpp) against oracle/flowvis_ref.py, known answers
derived by hand from the colour wheel, and inputs with NaN and inf.  GPU: the same through ops.flow_to_color, the video
predictor's CUDA graph (both network classes, the cascade captured for the first time) against the eager chain, and the
command line on a small video and an image pair.
"""
import ctypes
import importlib.util
import os

import numpy as np
import pytest
import torch

from maskflownet_b200 import MaskflowError, network, ops
from maskflownet_b200.video import VideoFlowPredictor
from oracle import flowvis_ref

from launchcheck import fp64_references  # noqa: F401
from launchcheck.emu import build, ptr

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
WHITE = (255, 255, 255)


def _random_flow(rng, N, H, W, scale=5.0):
    return (rng.standard_normal((N, H, W, 2)) * scale).astype(np.float32)


def _check_against_oracle(rgb, rad_max, flow, max_radius, bgr):
    want, want_rad = flowvis_ref.flow_to_color(flow, max_radius=max_radius, bgr=bgr)
    diff = np.abs(rgb.astype(np.int32) - want.astype(np.int32))
    if max_radius is not None:   # the branch at radius 1 is a discontinuity: float32 and float64 may fall either side
        rad = np.sqrt((flow.astype(np.float64) ** 2).sum(-1)) / max_radius
        diff = diff[np.abs(rad - 1.0) > 1e-6]
    assert diff.max() <= 1, diff.max()
    assert np.abs(rad_max - want_rad).max() <= 1e-6 * np.abs(want_rad).max()


# ---------------------------------------------------------------------------------------------------------------
# CPU: the kernel source on the host
# ---------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    L = build(tmp_path_factory, "flowvis_emu")
    L.emu_flow_to_color.argtypes = [ctypes.c_void_p] * 3 + [ctypes.c_int] * 3 + [ctypes.c_float, ctypes.c_int]
    L.emu_wheel_taps.argtypes = [ctypes.c_float, ctypes.c_float] + [ctypes.c_void_p] * 3
    return L


def _emu_color(emu, flow, max_radius=None, bgr=False):
    flow = np.ascontiguousarray(flow, dtype=np.float32)
    N, H, W, _ = flow.shape
    rgb = np.full((N, H, W, 3), 7, np.uint8)
    rad = np.full(N, np.nan, np.float32)
    emu.emu_flow_to_color(ptr(flow), ptr(rgb), ptr(rad), N, H, W, 0.0 if max_radius is None else max_radius, int(bgr))
    return rgb, rad


def _gpu_color(flow, max_radius=None, bgr=False):
    rgb, rad = ops.flow_to_color(torch.from_numpy(np.ascontiguousarray(flow, dtype=np.float32)).cuda(), max_radius, bgr)
    return rgb.cpu().numpy(), rad.cpu().numpy()


@pytest.mark.parametrize("max_radius", [None, 4.0])
def test_kernel_source_matches_oracle_on_host(emu, max_radius):
    flow = _random_flow(np.random.default_rng(0), 3, 37, 53)
    flow[1] *= 0.01                                     # samples of very different magnitude
    rgb, rad = _emu_color(emu, flow, max_radius)
    _check_against_oracle(rgb, rad, flow, max_radius, False)
    if max_radius is not None:
        r = np.sqrt((flow.astype(np.float64) ** 2).sum(-1)) / max_radius
        assert (r > 1).mean() > 0.1 and (r <= 1).mean() > 0.1          # both sides of the rim are exercised
    bgr, rad_bgr = _emu_color(emu, flow, max_radius, bgr=True)
    assert np.array_equal(bgr, rgb[..., ::-1]) and np.array_equal(rad_bgr, rad)


def _known_answers(color):
    z = np.zeros((1, 5, 7, 2), np.float32)
    rgb, rad = color(z)
    assert (rgb == 255).all() and rad[0] == 0.0
    for uv, want in (((1.0, 0.0), (255, 0, 0)), ((0.0, 1.0), (255, 229, 0)), ((-1.0, 0.0), (0, 209, 255)),
                     ((0.0, -1.0), (88, 0, 255))):
        f = z.copy()
        f[0, 2, 3] = uv                                   # +0.0, not -0.0: the sign of the zero selects the wheel end
        rgb, rad = color(f)
        assert tuple(rgb[0, 2, 3]) == want, (uv, tuple(rgb[0, 2, 3]))
        rest = np.ones((5, 7), bool)
        rest[2, 3] = False
        assert (rgb[0][rest] == 255).all() and rad[0] == np.float32(1.0)
    f = z.copy()
    f[0, 1, 1] = (1.0, 0.0)
    rgb, rad = color(f, 0.5)                              # fixed scale, outside the unit circle: darkened
    assert tuple(rgb[0, 1, 1]) == (191, 0, 0) and tuple(rgb[0, 0, 0]) == WHITE and rad[0] == 0.5


def test_known_answers_on_host(emu):
    _known_answers(lambda f, r=None: _emu_color(emu, f, r))


def test_nan_and_inf_stay_inside_the_wheel_on_host(emu):
    k0, k1, fr = ctypes.c_int(), ctypes.c_int(), ctypes.c_float()
    special = [np.nan, np.inf, -np.inf, 0.0, -0.0, 1.0, -1.0, 1e-30, 3e38]
    for u in special:
        for v in special:
            emu.emu_wheel_taps(u, v, ctypes.byref(k0), ctypes.byref(k1), ctypes.byref(fr))
            assert 0 <= k0.value < 55 and 0 <= k1.value < 55, (u, v, k0.value, k1.value)
    flow = _random_flow(np.random.default_rng(1), 2, 9, 11)
    flow[0, 1, 2] = (np.nan, 1.0)
    flow[0, 3, 4] = (np.inf, -np.inf)
    flow[1, 5, 6] = (-np.inf, np.nan)
    for r in (None, 3.0):
        rgb, rad = _emu_color(emu, flow, r)
        assert rgb.shape == (2, 9, 11, 3)


# ---------------------------------------------------------------------------------------------------------------
# GPU: ops.flow_to_color
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("shape", [(3, 37, 53), (8, 436, 1024)])
@pytest.mark.parametrize("max_radius", [None, 4.0])
def test_flow_to_color_matches_oracle(shape, max_radius):
    flow = _random_flow(np.random.default_rng(2), *shape)
    flow[0] *= 0.01
    rgb, rad = _gpu_color(flow, max_radius)
    _check_against_oracle(rgb, rad, flow, max_radius, False)
    bgr, _ = _gpu_color(flow, max_radius, bgr=True)
    assert np.array_equal(bgr, rgb[..., ::-1])


@pytest.mark.gpu
def test_flow_to_color_known_answers_and_single_image():
    _known_answers(_gpu_color)
    flow = _random_flow(np.random.default_rng(3), 1, 20, 30)
    rgb, rad = ops.flow_to_color(torch.from_numpy(flow[0]).cuda())
    assert rgb.shape == (20, 30, 3) and rad.shape == ()
    want, want_rad = _gpu_color(flow)
    assert np.array_equal(rgb.cpu().numpy(), want[0]) and float(rad) == float(want_rad[0])


@pytest.mark.gpu
def test_flow_to_color_argument_errors():
    good = torch.zeros(2, 8, 8, 2, device="cuda")
    with pytest.raises(MaskflowError, match="CUDA"):
        ops.flow_to_color(good.cpu())
    with pytest.raises(MaskflowError, match="float32"):
        ops.flow_to_color(good.double())
    for bad in (torch.zeros(2, 8, 8, 3, device="cuda"), torch.zeros(2, 2, 8, 8, device="cuda"),
                torch.zeros(8, 2, device="cuda")):
        with pytest.raises(MaskflowError, match="flow_to_color"):
            ops.flow_to_color(bad)
    for r in (0.0, -1.0, float("inf"), float("nan")):
        with pytest.raises(MaskflowError, match="max_radius"):
            ops.flow_to_color(good, r)
    with pytest.raises(MaskflowError, match="forward-only"):
        ops.flow_to_color(good.clone().requires_grad_())


# ---------------------------------------------------------------------------------------------------------------
# GPU: the video predictor
# ---------------------------------------------------------------------------------------------------------------
def _model(cls):
    torch.manual_seed(7)
    return cls().cuda().eval()


def _frames(n, H=100, W=150, seed=4):
    return np.random.default_rng(seed).integers(0, 256, (n, H, W, 3), dtype=np.uint8)


@pytest.mark.gpu
@pytest.mark.parametrize("cls,max_radius,bgr", [(network.MaskFlownetS, None, False), (network.MaskFlownet, 8.0, True)])
@pytest.mark.usefixtures("fp64_references")
def test_video_predictor_graph_equals_eager_chain(cls, max_radius, bgr):
    """11 frames at batch 4: two full batches and one of 2 pairs.  Each result equals, bit for bit, network.predict +
    ops.flow_to_color run eagerly on the same 4-pair batch (the last one padded with the last frame), since the
    convolutions' split-K plan depends on the batch."""
    model = _model(cls)
    frames = _frames(11)
    B, resize = 4, (128, 192)
    pred = VideoFlowPredictor(model, batch=B, resize=resize, max_radius=max_radius, bgr=bgr, want_flow=True)
    got = list(pred.run(iter(frames)))
    assert len(got) == 10
    for k in range(3):
        idx = [min(B * k + j, 10) for j in range(B + 1)]
        x = torch.from_numpy(frames[idx]).permute(0, 3, 1, 2).contiguous().cuda()
        flow, _ = network.predict(model, x[:B], x[1:], resize)
        rgb, _ = ops.flow_to_color(flow, max_radius, bgr)
        for j in range(min(B, 10 - B * k)):
            g_rgb, g_flow = got[B * k + j]
            assert g_rgb.shape == (100, 150, 3) and g_rgb.dtype == np.uint8 and g_flow.shape == (100, 150, 2)
            assert np.array_equal(g_rgb, rgb[j].cpu().numpy()), (k, j)
            assert np.array_equal(g_flow, flow[j].cpu().numpy()), (k, j)
    again = list(pred.run(list(frames[:6])))              # the graph is replayed for a second video of the same size
    assert all(np.array_equal(a[0], b[0]) for a, b in zip(again, got[:4]))
    assert len(again) == 5


@pytest.mark.gpu
def test_video_predictor_short_videos_and_bad_frames():
    model = _model(network.MaskFlownetS)
    pred = VideoFlowPredictor(model, batch=4)
    frames = _frames(3, 64, 96)
    assert list(pred.run([])) == [] and list(pred.run(frames[:1])) == []
    out = list(pred.run(frames))
    assert len(out) == 2 and out[0].shape == (64, 96, 3)
    with pytest.raises(MaskflowError, match="size"):
        list(pred.run([frames[0], frames[1], np.zeros((64, 90, 3), np.uint8)]))
    with pytest.raises(MaskflowError, match="uint8"):
        list(pred.run([frames[0].astype(np.float32)]))
    with pytest.raises(MaskflowError, match="max_radius"):
        VideoFlowPredictor(model, max_radius=-1.0)


# ---------------------------------------------------------------------------------------------------------------
# GPU: the command line
# ---------------------------------------------------------------------------------------------------------------
def _cli():
    spec = importlib.util.spec_from_file_location("predict_new_data", os.path.join(ROOT, "tools", "predict_new_data.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.mark.gpu
def test_predict_new_data_video_and_image_pair(tmp_path):
    cv2 = pytest.importorskip("cv2")
    cli = _cli()
    model = _model(network.MaskFlownetS)
    H, W = 72, 104
    frames = _frames(6, H, W, seed=5)
    src = str(tmp_path / "in.avi")
    wr = cv2.VideoWriter(src, cv2.VideoWriter_fourcc(*"MJPG"), 12.0, (W, H))
    for f in frames:
        wr.write(f)
    wr.release()
    dst = str(tmp_path / "flow.avi")
    assert cli.predict_files(model, dst, video_filepath=src, batch=2, resize=(64, 128)) == 5
    cap = cv2.VideoCapture(dst)
    assert cap.get(cv2.CAP_PROP_FPS) == pytest.approx(12.0)
    n = 0
    while True:
        ok, fr = cap.read()
        if not ok:
            break
        assert fr.shape == (H, W, 3)
        n += 1
    cap.release()
    assert n == 5

    p1, p2, out = str(tmp_path / "a.png"), str(tmp_path / "b.png"), str(tmp_path / "flow.png")
    cv2.imwrite(p1, frames[0])
    cv2.imwrite(p2, frames[1])
    assert cli.predict_files(model, out, image_1=p1, image_2=p2) == 1
    img = cv2.imread(out)
    assert img.shape == (H, W, 3)
    x = torch.from_numpy(frames[:2]).permute(0, 3, 1, 2).contiguous().cuda()
    flow, _ = network.predict(model, x[:1], x[1:])
    rgb, _ = ops.flow_to_color(flow)
    assert np.array_equal(img[..., ::-1], rgb[0].cpu().numpy())     # the PNG holds standard (R,G,B) colours
