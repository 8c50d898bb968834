"""The opt-in bf16 inference mode (network inference_precision = "bf16", MFN_CONV_BF16): every 3x3 convolution of the
forward multiplies bf16-rounded operands once (hi x hi) and accumulates in fp32; the dense blocks' and the context
network's activations are stored as bf16 activations (one plane).

Every convolution launch of bf16 forwards is judged against float64 of the operands the kernel actually read: the hi
plane of a bf16 activation, or x.to(bfloat16) for fp32 input, and w.to(bfloat16).  Bound per element, S = |x| (*) |w| +
|b| on the rounded operands:
    |got - ref| <= 2^-20 S        plus 2^-8 |ref| where the output is stored as a bf16 activation.
The storage term is bf16's unit roundoff: 8 significant bits, round to nearest, |v - bf16(v)| <= 2^-8 |v| (reached
within a factor 2 by test_bf16_checker_separates_kernel_arithmetic_from_near_misses; 2^-9 would not hold).
The LeakyReLU slope is handled by launchcheck.bounds.judge.  Sensitivity: on one real launch of each kind the bound must
reject, by CONTROL_MARGIN, the fp32-accurate result (float64 of the unrounded operands) and one dropped tap.

The rest of the forward (correlation, warps, sampler, pre/post-processing) is the fp32 path, checked by
test_bench_shapes.py / test_serving_shapes.py; here those launches run unchecked.  Also here: the fp32 path is unchanged
by a bf16 forward in between, training ignores the setting, the graph-replayed predictors follow the setting bit for
bit, and the C ABI rejects the bit where the wgmma kernel would not run.
"""
import ctypes
import os
import subprocess
import sys
import time

import numpy as np
import pytest
import torch
import torch.nn.functional as tF

from maskflownet_b200 import _lib, network, ops, video

from launchcheck import fp64_references  # noqa: F401
from launchcheck.bounds import (CONTROL_MARGIN, EPS_S, _expected_convs, activate, bf16_bound, bf16_near_misses,
                                bf16_terms, channel_slopes, judge)
from launchcheck.inputs import _deterministic, _images_u8, _named_model, _same, named_init
from launchcheck.recorders import BF16Recorder

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ------------------------------------------------------------------------------------------------------------------
# CPU: the bound accepts the bf16 kernel's arithmetic and rejects its near misses
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("store", [False, True])
def test_bf16_checker_separates_kernel_arithmetic_from_near_misses(store):
    """dc_conv1 at level 2 (579 -> 128), small image, emulated in torch: bf16-rounded x and w, fp32 accumulation, bias,
    LeakyReLU (and, store=True, the output rounded to bf16 as a bf16 activation stores it).  It passes the bound; the
    fp32-accurate result and a dropped tap fail it by more than CONTROL_MARGIN."""
    g = torch.Generator().manual_seed(6)
    Cin, Cout, H, W = 579, 128, 10, 18
    a = torch.randn((1, Cin, H, W), generator=g)
    x = torch.where(a > 0, a, 0.1 * a)
    w = named_init("dc_conv1.weight", (Cout, Cin, 3, 3))
    b = named_init("dc_conv1.bias", (Cout,))
    xr, wr = x.bfloat16().float(), w.bfloat16().float()
    kern = tF.leaky_relu(tF.conv2d(xr, wr, padding=1) + b.view(1, -1, 1, 1), 0.1)
    if store:
        kern = kern.bfloat16().float()
    pre, S = bf16_terms(xr.double(), wr.double(), b.double())
    bound = bf16_bound(pre, S, 0 if store else None)
    sl = channel_slopes(Cout, 0.1)
    ratio, _ = judge(kern, pre, sl, bound, S)
    assert ratio <= 1.0, ratio
    for name, alt in bf16_near_misses(x.double(), w.double(), xr.double(), wr.double(), b.double()).items():
        got = activate(alt, sl)
        if store:
            got = got.float().bfloat16().double()
        r, _ = judge(got, pre, sl, bound, S)
        assert r >= CONTROL_MARGIN, (name, r)


def test_inference_precision_values():
    m = network.MaskFlownet()
    assert m.inference_precision == "fp32" and m.MaskFlownet_S.inference_precision == "fp32"
    m.inference_precision = "bf16"
    assert m.MaskFlownet_S.inference_precision == "bf16"
    with pytest.raises(_lib.MaskflowError):
        m.inference_precision = "fp16"
    assert m.inference_precision == "bf16"


# ------------------------------------------------------------------------------------------------------------------
# GPU: the recorder
# ------------------------------------------------------------------------------------------------------------------
RUNS = {   # run: (model class, batch, H, W, image seed, through network.predict)
    "fwd": (network.MaskFlownetS, 8, 448, 1024, 51, False),
    "cascade": (network.MaskFlownet, 4, 448, 1024, 52, False),   # bench.py's cascade batch: level 2 has a split-K tail
    "cascade8": (network.MaskFlownet, 8, 448, 1024, 56, False),  # tools/precision_bench.py's cascade batch
    "tiny": (network.MaskFlownetS, 1, 64, 64, 53, False),
    "tiny_cascade": (network.MaskFlownet, 1, 64, 64, 54, False),
    "kitti": (network.MaskFlownetS, 1, 375, 1242, 55, True),
}


@pytest.mark.gpu
@pytest.mark.parametrize("run", list(RUNS))
@pytest.mark.usefixtures("fp64_references")
def test_every_convolution_of_a_bf16_forward_against_float64(run, monkeypatch):
    cls, N, H, W, seed, via_predict = RUNS[run]
    t0 = time.perf_counter()
    rec = BF16Recorder(monkeypatch, run)
    model = _named_model(cls).eval()
    model.inference_precision = "bf16"
    u1, u2 = _images_u8(seed=seed, n=N, h=H, w=W)
    if via_predict:
        flow, _ = network.predict(model, u1, u2)
    else:
        flow = network.predict_flow(model, u1, u2)
    assert bool(torch.isfinite(flow).all())
    torch.cuda.synchronize()
    monkeypatch.undo()
    rec.report()
    print(f"{run}: {len(rec.rows)} launches checked in {time.perf_counter() - t0:.1f} s")
    assert not rec.failures, "\n".join(rec.failures)

    convs = [r for r in rec.rows if r["op"] in ("conv3x3_slices", "conv3x3_split")]
    assert len(convs) == _expected_convs("cascade" if cls is network.MaskFlownet else "fwd"), len(convs)
    if run not in ("tiny", "tiny_cascade"):   # at 64x64 the first launch of a kind may be on a 1x1 level, where a
        # dropped corner tap reads only padding and the correlation input is zero but for the centre displacement
        assert set(BF16Recorder.KINDS) <= set(rec.controls), sorted(rec.controls)
        for tag, (name, rs) in rec.controls.items():
            assert min(rs.values()) >= CONTROL_MARGIN, (tag, name, rs)
    kernels = {r["kernel"] for r in convs}
    print(f"{run}: kernel variants {sorted(kernels)}")
    assert any(",fold,bf16>" in k for k in kernels) and any("CoutP=128,bf16>" in k for k in kernels), kernels
    if run == "fwd":   # level 6: 196 channels, two 128-channel halves (the cascade at batch 4 splits those launches)
        assert "conv3x3_wgmma_kernel<CoutP=256,bf16>" in kernels, kernels
    if run in ("fwd", "cascade", "cascade8"):
        assert {1, 2, 4, 8, 16} <= {r["dil"] for r in convs if r["op"] == "conv3x3_split"}
    if run == "cascade":
        assert any(r["split_out"] and r["ws"] > 0 and r["H"] == 112 for r in convs), \
            "no split-K launch with bf16 output at level 2"


# ------------------------------------------------------------------------------------------------------------------
# GPU: isolation
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("cls", [network.MaskFlownetS, network.MaskFlownet])
def test_bf16_forward_leaves_the_fp32_path_unchanged(cls):
    model = _named_model(cls).eval()
    u1, u2 = _images_u8(seed=61, n=2, h=256, w=448)
    with _deterministic():
        f1 = network.predict_flow(model, u1, u2).clone()
        model.inference_precision = "bf16"
        fb = network.predict_flow(model, u1, u2).clone()
        model.inference_precision = "fp32"
        f2 = network.predict_flow(model, u1, u2).clone()
    assert torch.equal(f1, f2)
    assert bool(torch.isfinite(fb).all()) and not torch.equal(fb, f1)
    d = (fb - f1).abs()
    print(f"{cls.__name__}: bf16 vs fp32 flow: mean |d| {float(d.mean()):.3g} px, max {float(d.max()):.3g} px")


_TRAIN_SCRIPT = r"""
import sys, torch
from maskflownet_b200 import network
torch.use_deterministic_algorithms(True)
res = []
for prec in ("fp32", "bf16", "fp32"):
    torch.manual_seed(0)
    m = network.MaskFlownetS().cuda().train()
    m.inference_precision = prec
    g = torch.Generator().manual_seed(1)
    a = torch.randn((2, 3, 128, 192), generator=g).cuda()
    b = torch.randn((2, 3, 128, 192), generator=g).cuda()
    preds = m(a, b)[0]
    loss = sum(p.square().mean() for p in preds)
    loss.backward()
    res.append((loss.detach().cpu(), {k: p.grad.detach().cpu() for k, p in m.named_parameters()}))
(l0, g0), (l1, g1), (l2, g2) = res
assert torch.equal(l0, l1) and torch.equal(l0, l2), (l0, l1, l2)
bad = [k for k in g0 if not (torch.equal(g0[k], g1[k]) and torch.equal(g0[k], g2[k]))]
assert not bad, bad[:5]
print("identical", float(l0), len(g0))
"""


@pytest.mark.gpu
def test_training_step_ignores_the_inference_precision():
    """Loss and every gradient of a training forward + backward are bit-identical with inference_precision fp32, bf16
    and fp32 again, under torch.use_deterministic_algorithms(True) (CUBLAS_WORKSPACE_CONFIG as test_deterministic.py)."""
    env = dict(os.environ, CUBLAS_WORKSPACE_CONFIG=":4096:8", PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    flags = ["-s"] if sys.flags.no_user_site else []
    r = subprocess.run([sys.executable, *flags, "-c", _TRAIN_SCRIPT], env=env, cwd=ROOT, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    assert "identical" in r.stdout


@pytest.mark.gpu
@pytest.mark.parametrize("cls", [network.MaskFlownetS, network.MaskFlownet])
def test_flow_predictor_follows_the_precision(cls):
    """FlowPredictor in bf16 equals the eager bf16 forward bit for bit; switching the precision between calls switches
    the replayed graph (and back)."""
    model = _named_model(cls).eval()
    p = _images_u8(seed=62, n=2, h=256, w=448)
    with _deterministic():
        e32 = network.predict_flow(model, *p).clone()
        model.inference_precision = "bf16"
        e16 = network.predict_flow(model, *p).clone()
        assert not torch.equal(e16, e32)
        pred = network.FlowPredictor(model)
        _same(pred(*p), e16, "graph, bf16")
        model.inference_precision = "fp32"
        _same(pred(*p), e32, "graph, fp32 after bf16")
        model.inference_precision = "bf16"
        _same(pred(*p), e16, "graph, bf16 again")
        if cls is network.MaskFlownet:   # the head's precision set on its own is part of the graph's key too
            model.MaskFlownet_S.inference_precision = "fp32"
            mixed = network.predict_flow(model, *p).clone()
            assert not torch.equal(mixed, e16) and not torch.equal(mixed, e32)
            _same(pred(*p), mixed, "graph, cascade bf16 with an fp32 head")
        torch.cuda.synchronize()


_PIPE_TRAIN_SCRIPT = r"""
import numpy as np, torch
from maskflownet_b200 import augment, pipeline
g = np.random.default_rng(65)
n, orig, target = 2, (160, 224), (128, 192)
img1 = g.integers(0, 256, (n, 3) + orig, dtype=np.uint8)
img2 = g.integers(0, 256, (n, 3) + orig, dtype=np.uint8)
label = (g.standard_normal((n, 2) + orig) * 2).astype(np.float32)
res = {}
for prec in ("fp32", "bf16"):
    torch.manual_seed(0)
    pipe = pipeline.PipelineFlownet(network_class="MaskFlownet_S", precision=prec, deterministic=True)
    geo = augment.GeometryAugmentation(angle_range=(-17, 17), zoom_range=(0.5, 1 / 0.9), aspect_range=(0.9, 1 / 0.9),
                                       translation_range=0.1, target_shape=target, orig_shape=orig, batch_size=n,
                                       relative_angle=0.25, relative_scale=(0.96, 1 / 0.96), relative_translation=0.25, seed=3)
    col = augment.ColorAugmentation(contrast_range=(-0.4, 0.8), brightness_sigma=0.1, channel_range=(0.8, 1.4), batch_size=n,
                                    shape=target, noise_range=(0, 0.04), saturation=0.5, hue=0.5, seed=4)
    epe = [pipe.train_batch(img1, img2, label, geo, col)["epe"] for _ in range(2)]
    assert pipe.network.inference_precision == prec
    res[prec] = (epe, {k: v.detach().cpu() for k, v in pipe.network.state_dict().items()})
(e0, s0), (e1, s1) = res["fp32"], res["bf16"]
assert e0 == e1, (e0, e1)
bad = [k for k in s0 if not torch.equal(s0[k], s1[k])]
assert not bad, bad[:5]
print("identical", e0)
"""


@pytest.mark.gpu
def test_pipeline_precision_applies_to_inference_only():
    """PipelineFlownet(precision=...): do_batch_mx, do_batch and predict run the chosen precision (bit for bit the eager
    forward of the same weights in that precision), and two train_batch steps of a bf16 pipeline give the fp32
    pipeline's losses and parameters bit for bit (in a fresh process: CUBLAS_WORKSPACE_CONFIG, deterministic=True)."""
    from maskflownet_b200 import pipeline
    with pytest.raises(_lib.MaskflowError):
        pipeline.PipelineFlownet(network_class="MaskFlownet_S", precision="fp16")
    g = np.random.default_rng(66)
    img1 = g.integers(0, 256, (2, 3, 128, 192), dtype=np.uint8)
    img2 = g.integers(0, 256, (2, 3, 128, 192), dtype=np.uint8)
    a, b = torch.from_numpy(img1).cuda(), torch.from_numpy(img2).cuda()
    eager = {}
    with _deterministic(), torch.no_grad():
        for prec in ("fp32", "bf16"):
            torch.manual_seed(0)
            pipe = pipeline.PipelineFlownet(network_class="MaskFlownet_S", precision=prec)
            assert pipe.network.inference_precision == prec
            net = pipe.network.eval()
            x1, x2, _ = ops.preprocess(a, b, ops.padded_size(128, 192))
            eager[prec] = net(x1, x2)[0][-1].clone()
            _same(pipe.do_batch_mx(a, b)[0][-1], eager[prec], f"do_batch_mx {prec}")
            ref = ops.postprocess(eager[prec], 128, 192, flip_channels=False, is_flow=True).permute(0, 3, 1, 2)
            _same(pipe.do_batch(a, b)[0], ref, f"do_batch {prec}")
            net.inference_precision = "bf16" if prec == "fp32" else "fp32"   # predict() restores the pipeline's setting
            got = next(pipe.predict([img1[0].transpose(1, 2, 0)], [img2[0].transpose(1, 2, 0)], 1))[0]
            assert net.inference_precision == prec
            x1, x2, _ = ops.preprocess(a[:1], b[:1], ops.padded_size(128, 192))    # batch 1: predict's split-K plans
            ref1 = ops.postprocess(net(x1, x2)[0][-1], 128, 192, flip_channels=True, is_flow=True)
            _same(torch.from_numpy(got), ref1[0].cpu(), f"predict {prec}")
    assert not torch.equal(eager["fp32"], eager["bf16"])
    env = dict(os.environ, CUBLAS_WORKSPACE_CONFIG=":4096:8", PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    flags = ["-s"] if sys.flags.no_user_site else []
    r = subprocess.run([sys.executable, *flags, "-c", _PIPE_TRAIN_SCRIPT], env=env, cwd=ROOT, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-4000:]
    assert "identical" in r.stdout


@pytest.mark.gpu
def test_video_predictor_follows_the_precision():
    """VideoFlowPredictor's flows equal the eager chain (preprocess, network, postprocess) in each precision, and a
    precision switch between two videos changes them."""
    model = _named_model(network.MaskFlownetS).eval()
    g = np.random.default_rng(63)
    frames = [g.integers(0, 256, (128, 192, 3), dtype=np.uint8) for _ in range(4)]
    vp = video.VideoFlowPredictor(model, batch=3, want_flow=True)
    got = {}
    with _deterministic():
        for prec in ("bf16", "fp32"):
            model.inference_precision = prec
            flows = [f for _, f in vp.run(frames)]
            x = torch.as_tensor(np.stack(frames)).cuda().permute(0, 3, 1, 2).contiguous()
            with torch.no_grad():
                a, b, _ = ops.preprocess(x[:3], x[1:], ops.padded_size(128, 192))
                ref = ops.postprocess(model(a, b)[0][-1], 128, 192, flip_channels=True, is_flow=True).cpu()
            for j in range(3):
                _same(torch.as_tensor(flows[j]), ref[j], f"video {prec}, pair {j}")
            got[prec] = ref
    assert not torch.equal(got["bf16"], got["fp32"])


@pytest.mark.gpu
def test_bf16_pack_is_torch_rounding_with_zero_pad():
    g = torch.Generator().manual_seed(64)
    src = (torch.randn((2, 21, 9, 13), generator=g) * 100).cuda()
    src[0, 0, 0, :4] = torch.tensor([1.0 + 2 ** -8, 1.0 + 3 * 2 ** -8, -(1.0 + 2 ** -8), 3.0e38])
    act = ops.SplitAct(2, 37, 9, 13, "cuda", bf16=True)       # 6 groups: channels 37..47 are the buffer's pad
    act.buf.fill_(0x5A)
    act.pack(src, 16)
    torch.cuda.synchronize()
    hi, lo = act.hi_lo()
    assert torch.equal(hi[:, 16:37], src.bfloat16().float()) and not bool(lo.any())
    ties = torch.tensor([1.0, 1.0 + 2 ** -6, -1.0])                          # round to nearest, ties to even
    assert torch.equal(hi[0, 16, 0, :3].cpu(), ties) and float(hi[0, 16, 0, 3]) == float(torch.tensor(3.0e38).bfloat16())
    raw = act.buf.view(torch.int16).view(2, 1, 6, 9, 13, 8).permute(0, 1, 2, 5, 3, 4).reshape(2, 48, 9, 13)
    assert not bool(raw[:, 37:48].any())                                     # pad channels of the slice are zero
    assert bool((act.buf.view(2, 6, 9, 13, 16)[:, :2] == 0x5A).all())        # channels 0..15 untouched


@pytest.mark.gpu
def test_bf16_bit_is_refused_where_the_wgmma_kernel_does_not_run():
    x = torch.randn((1, 16, 8, 32), device="cuda")
    w = torch.randn((16, 16, 3, 3), device="cuda")
    packed = ops.conv3x3_pack(w)
    out = torch.empty((1, 16, 8, 32), device="cuda")
    L = _lib.lib()
    args = [ctypes.c_void_p(x.data_ptr()), 0, ctypes.c_void_p(packed.data_ptr()), None, ctypes.c_void_p(out.data_ptr()), 0,
            1, 16, 8, 32, 16, 1, 1, ops.MFN_CONV_BF16, 0.1, None]
    try:
        _lib.set_tuning("conv_wgmma", 0)
        assert L.mfn_conv3x3_forward_ex(*args) == -2                          # MFN_ERR_UNSUPPORTED
    finally:
        _lib.set_tuning("conv_wgmma", 1)
    assert L.mfn_conv3x3_forward_ex(*args) == 0
    torch.cuda.synchronize()
    ref = tF.leaky_relu(tF.conv2d(x.bfloat16().double(), w.bfloat16().double(), padding=1), 0.1)
    assert float((out.double() - ref).abs().max()) <= EPS_S * float(tF.conv2d(x.abs().double(), w.abs().double(), padding=1).max())
    act32 = ops.SplitAct(1, 16, 8, 32, "cuda")
    act16 = ops.SplitAct(1, 16, 8, 32, "cuda", bf16=True)
    with pytest.raises(_lib.MaskflowError, match="bf16"):
        ops.conv3x3_split(act32, 0, 16, packed, None, 16, out=out, bf16=True)
    with pytest.raises(_lib.MaskflowError, match="bf16"):
        ops.conv3x3_split(act16, 0, 16, packed, None, 16, out=out)
    with pytest.raises(_lib.MaskflowError, match="bf16"):
        ops.conv3x3_split(act16, 0, 16, packed, None, 16, out_split=act32, bf16=True)
