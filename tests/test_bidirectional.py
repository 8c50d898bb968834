"""Bidirectional flow with forward-backward occlusion masks: the consistency kernel (csrc/consistency.cu,
ops.flow_consistency), the bidirectional forward of both networks (network.predict_bidirectional), the bidirectional
video predictor and `predict_new_data.py --occlusion`.

CPU: the kernel source compiled for the host (tests/host_emu/consistency_emu.cpp) against the float64 restatement of the
rule below (consistency_ref), known answers, and the C entry point's argument errors.  GPU: the same through
ops.flow_consistency; predict_bidirectional against two network.predict calls, direction by direction, within the
network-level tolerance of DESIGN.md section 2, with two controls that must fail it; the video predictor's graph against
the same chain run eagerly; the command line; the bf16 mode.

Ambiguous pixels (where float32 and float64 may decide differently) are excluded from the oracle comparisons and counted:
|d^2 - (alpha m^2 + beta)| <= 1e-4 (d^2 + alpha m^2 + beta), or a target within 1e-3 of a frame bound.  The oracle takes
the target x + u as the float32 sum the rule defines; everything after it is float64.
"""
import ctypes
import importlib.util
import os

import numpy as np
import pytest
import torch

from maskflownet_b200 import MaskflowError, _lib, network, ops
from maskflownet_b200.video import VideoFlowPredictor

from launchcheck.bidirectional import ALPHA, AMBIGUOUS_MAX, BETA, consistency_ref
from launchcheck.emu import build, ptr
from launchcheck.inputs import _deterministic

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
# DESIGN.md section 2, network level: 2e-3 px on flows of about 12 px, i.e. 1e-4 of the x20 flow scale.  A forward's
# rounding error grows with its activations, so flows larger than 12 px (random-init weights) scale the bound with them.
FLOW_TOL, FLOW_TOL_AT_PX = 1e-4 * 20.0, 12.0


def _flow_tol(*refs):
    return FLOW_TOL * max(1.0, max(float(r.abs().max()) for r in refs) / FLOW_TOL_AT_PX)


# ---------------------------------------------------------------------------------------------------------------
# the comparison with the float64 restatement of the rule (launchcheck/bidirectional.py)
# ---------------------------------------------------------------------------------------------------------------
def _compare(got_fw, got_bw, flow_fw, flow_bw, alpha=ALPHA, beta=BETA):
    """Masks against the oracle outside the ambiguous pixels; returns (excluded, compared) pixel counts."""
    occ_fw, occ_bw, amb_fw, amb_bw = consistency_ref(flow_fw, flow_bw, alpha, beta)
    excluded = 0
    for got, want, amb, nm in ((got_fw, occ_fw, amb_fw, "fw"), (got_bw, occ_bw, amb_bw, "bw")):
        assert got.dtype == np.uint8 and got.shape == want.shape and set(np.unique(got)) <= {0, 1}, nm
        bad = (got.astype(bool) != want) & ~amb
        assert not bad.any(), f"{nm}: {int(bad.sum())} pixels differ, first at {np.argwhere(bad)[0]}"
        excluded += int(amb.sum())
    return excluded, 2 * want.size


def _flows(rng, N, H, W):
    """Pairs that exercise every branch: near-consistent translations (both sides of the threshold), large random flows
    (targets anywhere, many outside the frame), targets in the last column / row cell (the x1 / y1 clamp), NaN and inf."""
    t = rng.uniform(-0.3, 0.3, (N, 1, 1, 2)) * np.array([W, H])
    fw = t + rng.normal(0, 0.4, (N, H, W, 2))
    bw = -t + rng.normal(0, 0.4, (N, H, W, 2))
    y, x = np.mgrid[0:H, 0:W]
    for f in (fw, bw):
        m = rng.random((N, H, W)) < 0.1
        f[m] = rng.normal(0, max(H, W), (int(m.sum()), 2))
        m = rng.random((N, H, W)) < 0.05
        f[..., 0] = np.where(m, (W - 1) - x - rng.uniform(0.01, 0.99, (N, H, W)), f[..., 0])
        m = rng.random((N, H, W)) < 0.05
        f[..., 1] = np.where(m, (H - 1) - y - rng.uniform(0.01, 0.99, (N, H, W)), f[..., 1])
        m = rng.random((N, H, W, 2)) < 0.01
        f[m] = rng.choice([np.nan, np.inf, -np.inf], int(m.sum()))
    return fw.astype(np.float32), bw.astype(np.float32)


def _known_answers(consistency):
    """consistency(flow_fw, flow_bw, alpha, beta) -> (occ_fw, occ_bw) as numpy, on (N,H,W,2) float32."""
    N, H, W = 2, 9, 13
    z = np.zeros((N, H, W, 2), np.float32)
    fw, bw = consistency(z, z, ALPHA, BETA)
    assert not fw.any() and not bw.any()
    y, x = np.mgrid[0:H, 0:W]

    def leaves(t):
        return ~((x + t[0] >= 0) & (x + t[0] <= W - 1) & (y + t[1] >= 0) & (y + t[1] <= H - 1))

    # integer translations land exactly on the last row / column (the x1 / y1 clamp) and on the first
    for t in ((2.5, -1.25), (1.0, 0.0), (0.0, -1.0), (-3.0, 2.0), (0.25, 0.5), (0.125, -0.25), (-12.0, 8.0), (13.0, 0.0)):
        f = np.broadcast_to(np.array(t, np.float32), z.shape).copy()
        fw, bw = consistency(f, -f, ALPHA, BETA)     # consistent: visible exactly where the target stays in the frame
        assert np.array_equal(fw, np.broadcast_to(leaves(t), fw.shape).astype(np.uint8)), t
        assert np.array_equal(bw, np.broadcast_to(leaves((-t[0], -t[1])), bw.shape).astype(np.uint8)), t
        for alpha, beta in ((ALPHA, BETA), (0.3, 0.1)):
            t2 = t[0] ** 2 + t[1] ** 2
            occluded = 4 * t2 > 2 * alpha * t2 + beta   # backward flow +t: d^2 = 4|t|^2, m^2 = 2|t|^2
            fw, bw = consistency(f, f.copy(), alpha, beta)   # the same flow both ways: both directions alike
            want = np.broadcast_to(leaves(t) | occluded, fw.shape).astype(np.uint8)
            assert np.array_equal(fw, want) and np.array_equal(bw, want), (t, alpha, beta)


# ---------------------------------------------------------------------------------------------------------------
# CPU: the kernel source on the host
# ---------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    L = build(tmp_path_factory, "consistency_emu")
    L.emu_flow_consistency.argtypes = [ctypes.c_void_p] * 4 + [ctypes.c_int] * 3 + [ctypes.c_float] * 2
    return L


def _emu_consistency(emu, flow_fw, flow_bw, alpha=ALPHA, beta=BETA):
    fw = np.ascontiguousarray(flow_fw, np.float32)
    bw = np.ascontiguousarray(flow_bw, np.float32)
    N, H, W, _ = fw.shape
    occ_fw = np.full((N, H, W), 7, np.uint8)
    occ_bw = np.full((N, H, W), 7, np.uint8)
    emu.emu_flow_consistency(ptr(fw), ptr(bw), ptr(occ_fw), ptr(occ_bw), N, H, W, alpha, beta)
    return occ_fw, occ_bw


def test_kernel_source_matches_oracle_on_host(emu):
    rng = np.random.default_rng(0)
    excluded = total = 0
    for shape in ((3, 37, 53), (1, 1, 1), (2, 1, 61), (2, 47, 1), (1, 2, 2), (4, 64, 96)):
        fw, bw = _flows(rng, *shape)
        occ_fw, occ_bw = _emu_consistency(emu, fw, bw)
        e, n = _compare(occ_fw, occ_bw, fw, bw)
        excluded, total = excluded + e, total + n
        if shape == (4, 64, 96):   # the flows reach both decisions inside the frame
            ref_fw = consistency_ref(fw, bw)[0]
            assert 0.2 < ref_fw.mean() < 0.8, ref_fw.mean()
    assert excluded <= AMBIGUOUS_MAX * total, (excluded, total)
    fw, bw = _flows(rng, 2, 20, 30)
    e, n = _compare(*_emu_consistency(emu, fw, bw, 0.2, 1.5), fw, bw, 0.2, 1.5)
    assert e <= AMBIGUOUS_MAX * n, (e, n)


def test_known_answers_on_host(emu):
    _known_answers(lambda f, b, alpha, beta: _emu_consistency(emu, f, b, alpha, beta))


def test_nan_and_inf_on_host(emu):
    z = np.zeros((1, 4, 5, 2), np.float32)
    for val in (np.nan, np.inf, -np.inf):
        for k in (0, 1):
            f = z.copy()
            f[0, 1, 2, k] = val                     # the pixel's own flow: its target fails every bound test
            fw, bw = _emu_consistency(emu, f, z)
            assert fw[0, 1, 2] == 1 and fw.sum() == 1, (val, k)
    for val in (np.nan, np.inf, -np.inf):           # a non-finite flow sampled by the other direction fails the test,
        f = z.copy()                                # at the corner itself and where it has weight 0 (NaN = inf * 0)
        f[0, 2, 3] = (0.0, val)
        fw, bw = _emu_consistency(emu, z, f)
        assert fw[0, 2, 3] == 1 and fw[0, 2, 2] == 1 and fw[0, 1, 3] == 1 and fw[0, 1, 2] == 1, val
        assert fw.sum() == 4 and bw[0, 2, 3] == 1 and bw.sum() == 1, val


def test_argument_errors_need_no_gpu():
    L = _lib.lib()
    buf = (ctypes.c_float * 64)()
    p = ctypes.cast(buf, ctypes.c_void_p)
    odd = ctypes.c_void_p(p.value + 4)
    f = L.mfn_flow_consistency
    assert f(None, p, p, p, 1, 2, 2, 0.01, 0.5, None) == -1 and b"null pointer" in L.mfn_last_error()
    assert f(p, p, p, None, 1, 2, 2, 0.01, 0.5, None) == -1 and b"null pointer" in L.mfn_last_error()
    for N, H, W in ((0, 2, 2), (1, 0, 2), (1, 2, -1)):
        assert f(p, p, p, p, N, H, W, 0.01, 0.5, None) == -1 and b"extent" in L.mfn_last_error()
    assert f(odd, p, p, p, 1, 2, 2, 0.01, 0.5, None) == -1 and b"aligned" in L.mfn_last_error()
    assert f(p, odd, p, p, 1, 2, 2, 0.01, 0.5, None) == -1 and b"aligned" in L.mfn_last_error()
    for alpha, beta in ((-0.01, 0.5), (0.01, -1.0), (float("nan"), 0.5), (0.01, float("inf")), (float("inf"), 0.5)):
        assert f(p, p, p, p, 1, 2, 2, alpha, beta, None) == -1 and b"alpha" in L.mfn_last_error(), (alpha, beta)


# ---------------------------------------------------------------------------------------------------------------
# GPU: ops.flow_consistency
# ---------------------------------------------------------------------------------------------------------------
def _gpu_consistency(flow_fw, flow_bw, alpha=ALPHA, beta=BETA):
    fw, bw = (torch.from_numpy(np.ascontiguousarray(a, np.float32)).cuda() for a in (flow_fw, flow_bw))
    occ_fw, occ_bw = ops.flow_consistency(fw, bw, alpha, beta)
    return occ_fw.cpu().numpy(), occ_bw.cpu().numpy()


@pytest.mark.gpu
@pytest.mark.parametrize("shape", [(3, 37, 53), (8, 436, 1024)])
def test_flow_consistency_matches_oracle(shape):
    fw, bw = _flows(np.random.default_rng(1), *shape)
    e, n = _compare(*_gpu_consistency(fw, bw), fw, bw)
    assert e <= AMBIGUOUS_MAX * n, (e, n)


@pytest.mark.gpu
def test_flow_consistency_known_answers_and_single_pair():
    _known_answers(_gpu_consistency)
    fw, bw = _flows(np.random.default_rng(2), 1, 20, 30)
    got = ops.flow_consistency(torch.from_numpy(fw[0]).cuda(), torch.from_numpy(bw[0]).cuda())
    want = _gpu_consistency(fw, bw)
    assert got[0].shape == (20, 30) and got[0].dtype == torch.uint8
    assert np.array_equal(got[0].cpu().numpy(), want[0][0]) and np.array_equal(got[1].cpu().numpy(), want[1][0])


@pytest.mark.gpu
def test_flow_consistency_argument_errors():
    good = torch.zeros(2, 8, 8, 2, device="cuda")
    with pytest.raises(MaskflowError, match="CUDA"):
        ops.flow_consistency(good.cpu(), good)
    with pytest.raises(MaskflowError, match="CUDA"):
        ops.flow_consistency(good, good.cpu())
    with pytest.raises(MaskflowError, match="float32"):
        ops.flow_consistency(good.double(), good)
    with pytest.raises(MaskflowError, match="contiguous"):
        ops.flow_consistency(good.transpose(1, 2), good)
    for bad in (torch.zeros(2, 8, 8, 3, device="cuda"), torch.zeros(8, 2, device="cuda")):
        with pytest.raises(MaskflowError, match="flow_consistency"):
            ops.flow_consistency(bad, bad)
    with pytest.raises(MaskflowError, match="differ"):
        ops.flow_consistency(good, torch.zeros(2, 8, 9, 2, device="cuda"))
    for alpha, beta in ((-0.01, 0.5), (0.01, -1.0), (float("nan"), 0.5), (0.01, float("inf"))):
        with pytest.raises(MaskflowError, match="alpha"):
            ops.flow_consistency(good, good, alpha, beta)
    with pytest.raises(MaskflowError, match="forward-only"):
        ops.flow_consistency(good.clone().requires_grad_(), good)


# ---------------------------------------------------------------------------------------------------------------
# GPU: predict_bidirectional
# ---------------------------------------------------------------------------------------------------------------
def _model(cls):
    torch.manual_seed(7)
    return cls().cuda().eval()


def _pairs(n, H, W, seed):
    g = np.random.default_rng(seed)
    a, b = (torch.from_numpy(g.integers(0, 256, (n, 3, H, W), dtype=np.uint8)).cuda() for _ in range(2))
    return a, b


def _flow_err(got, ref):
    return float((got - ref).abs().nan_to_num(float("inf")).max())


CASES = [(network.MaskFlownetS, 1, 64, 64), (network.MaskFlownetS, 8, 448, 1024), (network.MaskFlownetS, 1, 375, 1242),
         (network.MaskFlownet, 1, 64, 64), (network.MaskFlownet, 4, 448, 1024), (network.MaskFlownet, 1, 375, 1242)]


@pytest.mark.gpu
@pytest.mark.parametrize("cls,n,H,W", CASES, ids=[f"{c.__name__}-{n}x{h}x{w}" for c, n, h, w in CASES])
def test_predict_bidirectional_equals_two_predicts(cls, n, H, W, monkeypatch):
    """Under torch.use_deterministic_algorithms(True), so that both sides get bit-identical network inputs (the default
    preprocess sums with atomics) and what differs is the batch of 2N alone (its split-K plans)."""
    model = _model(cls)
    a, b = _pairs(n, H, W, seed=H + n)
    with _deterministic():
        fw, bw, occ_fw, occ_bw = network.predict_bidirectional(model, a, b)
        ref_fw, _ = network.predict(model, a, b)
        ref_bw, _ = network.predict(model, b, a)
        assert fw.shape == (n, H, W, 2) and bw.shape == (n, H, W, 2) and occ_fw.shape == (n, H, W)
        assert bool(torch.isfinite(ref_fw).all()) and bool(torch.isfinite(ref_bw).all())
        e_fw, e_bw = _flow_err(fw, ref_fw), _flow_err(bw, ref_bw)
        tol = _flow_tol(ref_fw, ref_bw)
        print(f"{cls.__name__} {n}x{H}x{W}: bound {tol:.3g} px, |fw - predict(a,b)| {e_fw:.3g}, |bw - predict(b,a)| "
              f"{e_bw:.3g}, occluded {float(occ_fw.float().mean()):.3f} / {float(occ_bw.float().mean()):.3f}")
        assert e_fw <= tol and e_bw <= tol, (e_fw, e_bw, tol)
        want_fw, want_bw = ops.flow_consistency(fw, bw)
        assert torch.equal(occ_fw, want_fw) and torch.equal(occ_bw, want_bw)
        # controls: the backward half computed as (a -> b), and no swap of the second images' features (c2 = c1)
        assert _flow_err(ref_fw, ref_bw) > 10 * tol
        monkeypatch.setattr(network, "_swap_halves", lambda t, k: t.clone())
        nfw, nbw, _, _ = network.predict_bidirectional(model, a, b)
        assert _flow_err(nfw, ref_fw) > 10 * tol and _flow_err(nbw, ref_bw) > 10 * tol


@pytest.mark.gpu
def test_bidirectional_forward_refuses_autograd():
    model = _model(network.MaskFlownetS)
    a, b = (torch.randn(1, 3, 64, 64, device="cuda") for _ in range(2))
    with pytest.raises(MaskflowError, match="inference"):
        model(a, b, bidirectional=True)
    with pytest.raises(MaskflowError, match="inference"):
        _model(network.MaskFlownet)(a, b, bidirectional=True)


@pytest.mark.gpu
@pytest.mark.parametrize("cls", [network.MaskFlownetS, network.MaskFlownet])
def test_predict_bidirectional_bf16(cls):
    """In bf16 mode every stored activation may carry bf16's rounding (test_bf16_mode.py's 2^-8 |ref| storage term), and
    the batch of 2N changes which values round which way.  Each direction must stay within the mode's own deviation
    from the fp32-accurate flow of the same pair: no further from network.predict in bf16 than the bf16 mode itself
    is from fp32."""
    model = _model(cls)
    a, b = _pairs(2, 128, 192, seed=9)
    ref32 = [network.predict(model, a, b)[0], network.predict(model, b, a)[0]]
    model.inference_precision = "bf16"
    fw, bw, occ_fw, occ_bw = network.predict_bidirectional(model, a, b)
    ref16 = [network.predict(model, a, b)[0], network.predict(model, b, a)[0]]
    for got, r16, r32, nm in ((fw, ref16[0], ref32[0], "fw"), (bw, ref16[1], ref32[1], "bw")):
        err, mode = _flow_err(got, r16), _flow_err(r16, r32)
        print(f"{cls.__name__} bf16 {nm}: max |flow| {float(r32.abs().max()):.3g} px, |bidirectional - predict| "
              f"{err:.3g}, |bf16 - fp32| {mode:.3g}")
        assert bool(torch.isfinite(got).all()) and 0 < mode and err <= mode, (nm, err, mode)
    want_fw, want_bw = ops.flow_consistency(fw, bw)
    assert torch.equal(occ_fw, want_fw) and torch.equal(occ_bw, want_bw)


# ---------------------------------------------------------------------------------------------------------------
# GPU: the video predictor
# ---------------------------------------------------------------------------------------------------------------
def _frames(n, H, W, seed):
    return np.random.default_rng(seed).integers(0, 256, (n, H, W, 3), dtype=np.uint8)


@pytest.mark.gpu
@pytest.mark.parametrize("cls,max_radius,bgr", [(network.MaskFlownetS, None, False), (network.MaskFlownet, 8.0, True)])
def test_video_predictor_bidirectional_graph_equals_eager_chain(cls, max_radius, bgr):
    """7 frames at batch 4 (one full batch and one of 2 pairs), then a 3-frame video (2 pairs, shorter than one batch):
    every output equals, bit for bit, predict_bidirectional + ops.flow_to_color run eagerly on the same 4-pair batch (the
    last one padded with the last frame), and the forward flows equal bidirectional=False's within the network-level
    tolerance."""
    model = _model(cls)
    B, resize, H, W = 4, (128, 192), 100, 150
    with _deterministic():
        pred = VideoFlowPredictor(model, batch=B, resize=resize, max_radius=max_radius, bgr=bgr, want_flow=True,
                                  bidirectional=True)
        short = VideoFlowPredictor(model, batch=B, resize=resize, max_radius=max_radius, bgr=bgr, bidirectional=True)
        plain = VideoFlowPredictor(model, batch=B, resize=resize, want_flow=True)
        for frames in (_frames(7, H, W, seed=4), _frames(3, H, W, seed=5)):
            T = len(frames) - 1
            got = list(pred.run(iter(frames)))
            got_short = list(short.run(list(frames)))
            one_way = [f for _, f in plain.run(list(frames))]
            assert len(got) == T and len(got_short) == T and len(one_way) == T
            for k in range((T + B - 1) // B):
                idx = [min(B * k + j, T) for j in range(B + 1)]
                x = torch.from_numpy(frames[idx]).permute(0, 3, 1, 2).contiguous().cuda()
                fw, bw, occ_fw, occ_bw = network.predict_bidirectional(model, x[:B], x[1:], resize)
                rgb, _ = ops.flow_to_color(fw, max_radius, bgr)
                for j in range(min(B, T - B * k)):
                    t = B * k + j
                    g_rgb, g_fw, g_bw, g_ofw, g_obw = got[t]
                    assert g_rgb.shape == (H, W, 3) and g_fw.shape == (H, W, 2) and g_ofw.shape == (H, W)
                    assert g_ofw.dtype == np.uint8 and g_obw.dtype == np.uint8
                    for g, e, nm in ((g_rgb, rgb, "rgb"), (g_fw, fw, "flow"), (g_bw, bw, "flow_bw"),
                                     (g_ofw, occ_fw, "occ_fw"), (g_obw, occ_bw, "occ_bw")):
                        assert np.array_equal(g, e[j].cpu().numpy()), (len(frames), t, nm)
                    s_rgb, s_ofw, s_obw = got_short[t]
                    assert np.array_equal(s_rgb, g_rgb) and np.array_equal(s_ofw, g_ofw) and np.array_equal(s_obw, g_obw)
                    err = float(np.abs(g_fw - one_way[t]).max())
                    tol = _flow_tol(torch.from_numpy(one_way[t]))
                    assert err <= tol, (len(frames), t, err, tol)


# ---------------------------------------------------------------------------------------------------------------
# GPU: the command line
# ---------------------------------------------------------------------------------------------------------------
def _cli():
    spec = importlib.util.spec_from_file_location("predict_new_data", os.path.join(ROOT, "tools", "predict_new_data.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.mark.gpu
def test_predict_new_data_writes_occlusion(tmp_path):
    cv2 = pytest.importorskip("cv2")
    cli = _cli()
    model = _model(network.MaskFlownetS)
    H, W = 72, 104
    frames = _frames(5, H, W, seed=6)
    p1, p2 = str(tmp_path / "a.png"), str(tmp_path / "b.png")
    cv2.imwrite(p1, frames[0])
    cv2.imwrite(p2, frames[1])
    out, occ = str(tmp_path / "flow.png"), str(tmp_path / "occ.png")
    assert cli.predict_files(model, out, image_1=p1, image_2=p2, occlusion_filepath=occ) == 1
    mask = cv2.imread(occ, cv2.IMREAD_UNCHANGED)
    assert mask.shape == (H, W) and mask.dtype == np.uint8 and set(np.unique(mask)) <= {0, 255}
    x = torch.from_numpy(frames[:2]).permute(0, 3, 1, 2).contiguous().cuda()
    fw, _, occ_fw, _ = network.predict_bidirectional(model, x[:1], x[1:])
    assert np.array_equal(mask, occ_fw[0].cpu().numpy() * 255)
    rgb, _ = ops.flow_to_color(fw)
    assert np.array_equal(cv2.imread(out)[..., ::-1], rgb[0].cpu().numpy())

    src = str(tmp_path / "in.avi")
    wr = cv2.VideoWriter(src, cv2.VideoWriter_fourcc(*"MJPG"), 10.0, (W, H))
    for f in frames:
        wr.write(f)
    wr.release()
    dst, occ_v = str(tmp_path / "flow.avi"), str(tmp_path / "occ.avi")
    assert cli.predict_files(model, dst, video_filepath=src, batch=2, resize=(64, 128), occlusion_filepath=occ_v) == 4
    for path in (dst, occ_v):
        cap = cv2.VideoCapture(path)
        assert cap.get(cv2.CAP_PROP_FPS) == pytest.approx(10.0)
        n = 0
        while True:
            ok, fr = cap.read()
            if not ok:
                break
            assert fr.shape[:2] == (H, W)
            n += 1
        cap.release()
        assert n == 4, path
