"""Backward of the image warp: GridGenerator('warp'), BilinearSampler and the fused cascade-input builder K5
(csrc/image_warp_bwd.cu, ops.grid_generator_warp / bilinear_sampler / reconstruction2d / image_warp_concat), and what it
enables: the MaskFlownet cascade trained end to end, with or without a frozen head.

CPU: the kernel source compiled for the host (tests/host_emu/image_warp_bwd_emu.cpp) against torch autograd, and the
argument checks of the three entry points.  GPU: the autograd Functions against oracle/torch_ref.py autograd on CUDA, the
cascade's training step against the same step with the K5 reference composition, and PipelineFlownet's cascade recipe.

The position gradient of bilinear sampling is discontinuous at integer sample positions, so the inputs are built with
fractional parts in [0.2, 0.8] (flows = multiples of 16 pixels + that fraction: the fraction survives Upsample(4), whose
taps are multiples of 1/4), and displacements of up to 32 pixels so that samples leave the image.
"""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as tF

from maskflownet_b200 import _lib
from oracle import torch_ref

from launchcheck import fp64_references  # noqa: F401
from launchcheck.emu import build, ptr


def _positions(rng, shape, lo, hi):
    """real sample coordinates in [lo, hi) whose fractional parts lie in [0.2, 0.8]"""
    return (rng.integers(lo, hi, shape) + rng.uniform(0.2, 0.8, shape)).astype(np.float64)


def _coarse_flow(rng, N, Hq, Wq, scale, kmax=1):
    """(N,2,Hq,Wq) flow_q such that Upsample(4)(flow_q) * scale = 16 * integer + a fraction in [0.2, 0.8] everywhere"""
    k = rng.integers(-kmax, kmax + 1, (N, 2, Hq, Wq))
    return ((16.0 * k + rng.uniform(0.2, 0.8, (N, 2, Hq, Wq))) / scale).astype(np.float32)


def _rel_err(got, want):
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    return np.abs(got - want).max() / max(np.abs(want).max(), 1e-6)


# ---------------------------------------------------------------------------------------------------------------
# CPU: the kernel source on the host
# ---------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    L = build(tmp_path_factory, "image_warp_bwd_emu")
    L.emu_image_warp_concat_backward.argtypes = [ctypes.c_void_p] * 7 + [ctypes.c_int] * 4 + [ctypes.c_float]
    return L


def test_kernel_source_bilinear_sampler_backward_on_host(emu):
    rng = np.random.default_rng(0)
    N, C, H, W, OH, OW = 2, 3, 12, 20, 9, 14
    data = rng.standard_normal((N, C, H, W)).astype(np.float32)
    xr, yr = _positions(rng, (N, OH, OW), -3, W + 2), _positions(rng, (N, OH, OW), -3, H + 2)
    grid = np.stack([xr / ((W - 1) / 2) - 1, yr / ((H - 1) / 2) - 1], axis=1).astype(np.float32)
    go = rng.standard_normal((N, C, OH, OW)).astype(np.float32)
    assert ((xr < 0) | (xr > W - 1) | (yr < 0) | (yr > H - 1)).mean() > 0.2          # samples leave the image
    d = torch.from_numpy(data).double().requires_grad_()
    g = torch.from_numpy(grid).double().requires_grad_()
    tF.grid_sample(d, g.permute(0, 2, 3, 1), mode="bilinear", padding_mode="zeros", align_corners=True).backward(
        torch.from_numpy(go).double())
    base = rng.standard_normal(data.shape).astype(np.float32)                           # accumulated into
    gd, gg = base.copy(), np.full_like(grid, np.nan)
    emu.emu_bilinear_sampler_backward(ptr(go), ptr(data), ptr(grid), ptr(gd), ptr(gg), N, C, H, W, OH, OW)
    assert _rel_err(gd - base, d.grad.numpy()) < 2e-5
    assert _rel_err(gg, g.grad.numpy()) < 2e-5
    gg2 = np.full_like(grid, np.nan)                                                    # grid only, data only
    emu.emu_bilinear_sampler_backward(ptr(go), ptr(data), ptr(grid), None, ptr(gg2), N, C, H, W, OH, OW)
    assert np.array_equal(gg, gg2)
    gd2 = np.zeros_like(data)
    emu.emu_bilinear_sampler_backward(ptr(go), ptr(data), ptr(grid), ptr(gd2), None, N, C, H, W, OH, OW)
    assert _rel_err(gd2, d.grad.numpy()) < 2e-5


def test_kernel_source_grid_generator_backward_on_host(emu):
    rng = np.random.default_rng(1)
    N, H, W = 2, 12, 20
    flow = torch.from_numpy(rng.standard_normal((N, 2, H, W))).requires_grad_()
    xs, ys = torch.arange(W, dtype=torch.float64).view(1, W), torch.arange(H, dtype=torch.float64).view(H, 1)
    grid = torch.stack([(flow[:, 0] + xs) / ((W - 1) / 2) - 1, (flow[:, 1] + ys) / ((H - 1) / 2) - 1], dim=1)
    gg = rng.standard_normal((N, 2, H, W)).astype(np.float32)
    grid.backward(torch.from_numpy(gg).double())
    gf = np.full_like(gg, np.nan)
    emu.emu_grid_generator_warp_backward(ptr(gg), ptr(gf), N, H, W)
    assert _rel_err(gf, flow.grad.numpy()) < 1e-6


def _k5_reference(im2, flow_up, mask_up, g40, scale):
    """torch autograd (float64) of c40 w.r.t. im2, the up-sampled flow and the up-sampled mask (leaves)"""
    i2 = torch.from_numpy(im2).double().requires_grad_()
    fu = torch.from_numpy(flow_up).double().requires_grad_()
    mu = torch.from_numpy(mask_up).double().requires_grad_()
    c40 = torch.cat([torch_ref.reconstruction2d(i2, fu * scale), torch.sigmoid(mu) - 0.5], dim=1)
    c40.backward(torch.from_numpy(g40).double())
    return i2.grad.numpy(), fu.grad.numpy(), mu.grad.numpy()


def test_kernel_source_image_warp_concat_backward_on_host(emu):
    rng = np.random.default_rng(2)
    N, Ci, H, W, scale = 2, 3, 12, 20, 20.0
    im2 = rng.random((N, Ci, H, W)).astype(np.float32)
    fq = _coarse_flow(rng, N, H // 4, W // 4, scale)
    mq = rng.standard_normal((N, 1, H // 4, W // 4)).astype(np.float32)
    g40 = rng.standard_normal((N, Ci + 1, H, W)).astype(np.float32)
    up = lambda a: torch_ref.upsample(torch.from_numpy(a).double(), 4).numpy()
    want_i2, want_fu, want_mu = _k5_reference(im2, up(fq), up(mq), g40, scale)
    pos = up(fq) * scale + np.stack(np.meshgrid(np.arange(H), np.arange(W), indexing="ij"))[None]
    assert ((pos[:, 0] < 0) | (pos[:, 0] > H - 1) | (pos[:, 1] < 0) | (pos[:, 1] > W - 1)).mean() > 0.2
    base = rng.standard_normal(im2.shape).astype(np.float32)
    gi2, gfu, gmu = base.copy(), np.full((N, 2, H, W), np.nan, np.float32), np.full((N, 1, H, W), np.nan, np.float32)
    emu.emu_image_warp_concat_backward(ptr(g40), ptr(im2), ptr(fq), ptr(mq), ptr(gi2), ptr(gfu), ptr(gmu),
                                       N, Ci, H, W, scale)
    assert _rel_err(gi2 - base, want_i2) < 2e-5
    assert _rel_err(gfu, want_fu) < 2e-5
    assert _rel_err(gmu, want_mu) < 1e-5
    for which in range(3):                       # each output alone gives the same numbers
        outs = [None, None, None]
        outs[which] = np.zeros_like((gi2, gfu, gmu)[which])
        emu.emu_image_warp_concat_backward(ptr(g40), ptr(im2), ptr(fq), ptr(mq), *[ptr(o) for o in outs], N, Ci, H, W,
                                           scale)
        want = (gi2 - base, gfu, gmu)[which]
        assert np.array_equal(outs[which], want) if which else _rel_err(outs[0], want) < 1e-6


def test_backward_argument_errors_need_no_gpu():
    L = _lib.lib()
    buf = (ctypes.c_float * 16)()
    p = ctypes.cast(buf, ctypes.c_void_p)
    assert L.mfn_grid_generator_warp_backward(None, p, 1, 4, 4, None) == -1 and b"null pointer" in L.mfn_last_error()
    assert L.mfn_grid_generator_warp_backward(p, p, 1, 1, 4, None) == -1 and b"H, W > 1" in L.mfn_last_error()
    assert L.mfn_bilinear_sampler_backward(p, None, p, p, p, 1, 1, 2, 2, 2, 2, None) == -1
    assert b"null pointer" in L.mfn_last_error()
    assert L.mfn_bilinear_sampler_backward(p, p, p, None, None, 1, 1, 2, 2, 2, 2, None) == -1
    assert b"null pointer" in L.mfn_last_error()
    assert L.mfn_bilinear_sampler_backward(p, p, p, p, p, 1, 1, 2, 2, 0, 2, None) == -1
    assert b"bad extent" in L.mfn_last_error()
    assert L.mfn_image_warp_concat_backward(p, p, None, p, p, p, p, 1, 3, 4, 4, 20.0, None) == -1
    assert b"null pointer" in L.mfn_last_error()
    assert L.mfn_image_warp_concat_backward(p, p, p, p, None, None, None, 1, 3, 4, 4, 20.0, None) == -1
    assert b"null pointer" in L.mfn_last_error()
    assert L.mfn_image_warp_concat_backward(p, p, p, p, None, p, p, 1, 3, 6, 8, 20.0, None) == -1
    assert b"multiples of 4" in L.mfn_last_error()
    assert L.mfn_image_warp_concat_backward(p, p, p, p, None, p, p, 1, 0, 4, 4, 20.0, None) == -1


# ---------------------------------------------------------------------------------------------------------------
# GPU: the autograd Functions
# ---------------------------------------------------------------------------------------------------------------
DEV = "cuda"


def _cu(a, grad=False):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV).requires_grad_(grad)


def _ref_on_cuda(fn, *args):
    """oracle/torch_ref.py builds its index tensors with the default device: evaluate it on the GPU in float64"""
    with torch.device(DEV):
        return fn(*args)


def _close(got, want, tol=1e-4):
    err = (got.double() - want.double()).abs().max().item()
    assert err <= tol * max(want.abs().max().item(), 1e-6), (err, want.abs().max().item())


@pytest.mark.gpu
def test_bilinear_sampler_grid_generator_reconstruction_autograd():
    from maskflownet_b200 import ops
    rng = np.random.default_rng(3)
    N, C, H, W = 2, 3, 24, 40
    img = rng.standard_normal((N, C, H, W)).astype(np.float32)
    flow_yx = np.stack([_positions(rng, (N, H, W), -6, 6), _positions(rng, (N, H, W), -6, 6)], axis=1).astype(np.float32)
    go = _cu(rng.standard_normal((N, C, H, W)).astype(np.float32))
    # reconstruction2d = GridGenerator + BilinearSampler, both differentiable
    x, f = _cu(img, True), _cu(flow_yx, True)
    out = ops.reconstruction2d(x, f)
    out.backward(go)
    xr, fr = _cu(img).double().requires_grad_(), _cu(flow_yx).double().requires_grad_()
    ref = _ref_on_cuda(torch_ref.reconstruction2d, xr, fr)
    ref.backward(go.double())
    _close(out.detach(), ref.detach())
    _close(x.grad, xr.grad)
    _close(f.grad, fr.grad)
    # the two operators separately: sampler w.r.t. data and grid, generator w.r.t. flow
    grid = ops.grid_generator_warp(_cu(flow_yx).flip(1).contiguous())
    d, g = _cu(img, True), grid.clone().requires_grad_()
    ops.bilinear_sampler(d, g).backward(go)
    dr, gr = _cu(img).double().requires_grad_(), grid.double().requires_grad_()
    tF.grid_sample(dr, gr.permute(0, 2, 3, 1), mode="bilinear", padding_mode="zeros", align_corners=True).backward(go.double())
    _close(d.grad, dr.grad)
    _close(g.grad, gr.grad)
    fl = _cu(flow_yx, True)
    gg = torch.randn(N, 2, H, W, device=DEV)
    ops.grid_generator_warp(fl).backward(gg)
    _close(fl.grad, torch.stack([gg[:, 0] / ((W - 1) / 2), gg[:, 1] / ((H - 1) / 2)], dim=1), 1e-6)
    # only the operand that requires grad gets one
    d2 = _cu(img, True)
    ops.bilinear_sampler(d2, grid).backward(go)
    _close(d2.grad, dr.grad)


def _k5_case(seed, N, Ci, H, W, scale=20.0):
    rng = np.random.default_rng(seed)
    im1 = rng.random((N, Ci, H, W)).astype(np.float32) - 0.5
    im2 = rng.random((N, Ci, H, W)).astype(np.float32) - 0.5
    fq = _coarse_flow(rng, N, H // 4, W // 4, scale, kmax=2)
    mq = rng.standard_normal((N, 1, H // 4, W // 4)).astype(np.float32)
    g30 = rng.standard_normal((N, Ci + 1, H, W)).astype(np.float32)
    g40 = rng.standard_normal((N, Ci + 1, H, W)).astype(np.float32)
    return im1, im2, fq, mq, g30, g40


@pytest.mark.gpu
@pytest.mark.parametrize("N,Ci,H,W", [(2, 3, 12, 20), (2, 3, 64, 96), (4, 3, 448, 1024)])
def test_image_warp_concat_autograd(N, Ci, H, W):
    from maskflownet_b200 import ops
    im1, im2, fq, mq, g30, g40 = _k5_case(4, N, Ci, H, W)
    a = [_cu(v, True) for v in (im1, im2, fq, mq)]
    c30, c40 = ops.image_warp_concat(*a, 20.0)
    torch.autograd.backward([c30, c40], [_cu(g30), _cu(g40)])
    r = [_cu(v).double().requires_grad_() for v in (im1, im2, fq, mq)]
    ref = _ref_on_cuda(torch_ref.image_warp_concat, r[1], r[2], r[3], 20.0)
    ref.backward(_cu(g40).double())
    _close(c40.detach(), ref.detach())
    assert torch.equal(a[0].grad, _cu(g30)[:, :Ci])
    for got, want in zip(a[1:], r[1:]):
        _close(got.grad, want.grad)
    # im2 that does not require grad gets none; flow and mask still get theirs
    b = [_cu(im1), _cu(im2), _cu(fq, True), _cu(mq, True)]
    _, c40b = ops.image_warp_concat(*b, 20.0, want_c30=False)
    c40b.backward(_cu(g40))
    assert b[1].grad is None and torch.equal(b[2].grad, a[2].grad) and torch.equal(b[3].grad, a[3].grad)


@pytest.mark.gpu
def test_image_warp_concat_backward_is_deterministic():
    from maskflownet_b200 import ops
    _, im2, fq, mq, _, g40 = _k5_case(5, 4, 3, 320, 768)
    grads = []
    for _ in range(2):
        f, m = _cu(fq, True), _cu(mq, True)
        ops.image_warp_concat(None, _cu(im2), f, m, 20.0, want_c30=False)[1].backward(_cu(g40))
        grads.append((f.grad, m.grad))
    assert torch.equal(grads[0][0], grads[1][0]) and torch.equal(grads[0][1], grads[1][1])


@pytest.mark.gpu
def test_image_warp_concat_without_grad_is_one_launch():
    from maskflownet_b200 import ops
    im1, im2, fq, mq, _, _ = _k5_case(6, 2, 3, 32, 48)
    a = [_cu(v, True) for v in (im1, im2, fq, mq)]
    n0 = _lib.launch_count()
    with torch.no_grad():
        c30, c40 = ops.image_warp_concat(*a, 20.0)
    assert _lib.launch_count() == n0 + 1 and _lib.last_kernel() == "image_warp_concat_kernel"
    assert c40.grad_fn is None and not c40.requires_grad
    n0 = _lib.launch_count()
    ops.image_warp_concat(*[v.detach() for v in a], 20.0)
    assert _lib.launch_count() == n0 + 1


# ---------------------------------------------------------------------------------------------------------------
# GPU: the cascade trained end to end
# ---------------------------------------------------------------------------------------------------------------
def _reference_image_warp_concat(im1, im2, flow_q, mask_q, scale=20.0, want_c30=True):
    """ops.image_warp_concat as the torch_ref composition (network/MaskFlownet.py:308-313), on the tensors' device"""
    with torch.device(im2.device):
        c40 = torch_ref.image_warp_concat(im2, flow_q, mask_q, scale)
    c30 = torch.cat([im1, torch.zeros_like(c40[:, -1:])], dim=1) if want_c30 else None
    return c30, c40


@pytest.mark.gpu
@pytest.mark.usefixtures("fp64_references")
def test_cascade_training_step_with_trainable_head(monkeypatch):
    """One MaskFlownet (cascade) training step with the S head trainable: every head parameter gets a finite, non-zero
    gradient through K5's backward, and the loss and all gradients equal the same step with K5 replaced by the torch_ref
    composition up to the criterion of the tensor-core training-step test (a swapped y/x or a missing x20 is O(1))."""
    from maskflownet_b200 import losses, network, ops
    torch.manual_seed(3)
    model = network.MaskFlownet().cuda().train()
    g = torch.Generator().manual_seed(5)
    a = torch.rand(2, 3, 128, 192, generator=g).cuda() - 0.5
    b = torch.rand(2, 3, 128, 192, generator=g).cuda() - 0.5
    flow = (torch.randn(2, 2, 128, 192, generator=g) * 2).cuda()
    mask = torch.ones(2, 1, 128, 192).cuda()

    def step():
        model.zero_grad(set_to_none=True)
        preds = model(a, b)[0]
        loss = losses.multiscale_epe(flow, mask, preds).sum()
        loss.backward()
        return loss.item(), {k: p.grad.clone() for k, p in model.named_parameters() if p.grad is not None}

    ours = step()
    head = dict(model.MaskFlownet_S.named_parameters())
    for k in head:
        gr = ours[1].get("MaskFlownet_S." + k)
        assert gr is not None and torch.isfinite(gr).all() and gr.abs().max() > 0, k
    monkeypatch.setattr(ops, "image_warp_concat", _reference_image_warp_concat)
    ref = step()
    assert abs(ours[0] - ref[0]) < 1e-4 * max(1.0, abs(ref[0])), (ours[0], ref[0])
    assert ours[1].keys() == ref[1].keys() and len(ours[1]) == len(list(model.parameters()))
    worst = max(((ours[1][k] - ref[1][k]).abs().max().item() / max(ref[1][k].abs().max().item(), 1e-6), k) for k in ref[1])
    assert worst[0] < 5e-2, worst


@pytest.mark.gpu
def test_pipeline_cascade_trains_with_and_without_fixed_head():
    """PipelineFlownet(network_class="MaskFlownet") with the real augmentation blocks: train_batch updates the head; after
    fix_head() (the reference recipe, main.py:133-139) a step leaves every head weight bitwise unchanged and updates the
    cascade."""
    from maskflownet_b200 import augment, pipeline
    rng = np.random.default_rng(7)
    n, orig, target = 2, (160, 224), (128, 192)
    pipe = pipeline.PipelineFlownet(network_class="MaskFlownet", lr_schedule=[(10, 1e-4)])
    geo = augment.GeometryAugmentation(angle_range=(-17, 17), zoom_range=(0.5, 1 / 0.9), aspect_range=(0.9, 1 / 0.9),
                                       translation_range=0.1, target_shape=target, orig_shape=orig, batch_size=n,
                                       relative_angle=0.25, relative_scale=(0.96, 1 / 0.96), relative_translation=0.25, seed=3)
    col = augment.ColorAugmentation(contrast_range=(-0.4, 0.8), brightness_sigma=0.1, channel_range=(0.8, 1.4), batch_size=n,
                                    shape=target, noise_range=(0, 0.04), saturation=0.5, hue=0.5, seed=4)
    img1 = rng.integers(0, 256, (n, 3) + orig, dtype=np.uint8)
    img2 = rng.integers(0, 256, (n, 3) + orig, dtype=np.uint8)
    label = (rng.standard_normal((n, 2) + orig) * 2).astype(np.float32)
    head, net = pipe.network.MaskFlownet_S, pipe.network
    w0 = head.conv1a.weight.detach().clone()
    out = pipe.train_batch(img1, img2, label, geo, col)
    assert np.isfinite(out["epe"]) and not torch.equal(head.conv1a.weight, w0)
    pipe.fix_head()
    before = {k: p.detach().clone() for k, p in head.named_parameters()}
    c0 = net.conv1x.weight.detach().clone()
    out = pipe.train_batch(img1, img2, label, geo, col)
    assert np.isfinite(out["epe"]) and not torch.equal(net.conv1x.weight, c0)
    assert all(torch.equal(p, before[k]) for k, p in head.named_parameters())


@pytest.mark.gpu
def test_mx_shim_image_warp_is_differentiable():
    from maskflownet_b200 import mx
    F = mx.nd
    rng = np.random.default_rng(8)
    N, C, H, W = 2, 3, 16, 24
    img = rng.standard_normal((N, C, H, W)).astype(np.float32)
    flow_xy = np.stack([_positions(rng, (N, H, W), -5, 5), _positions(rng, (N, H, W), -5, 5)], axis=1).astype(np.float32)
    go = rng.standard_normal((N, C, H, W)).astype(np.float32)
    data, flow = _cu(img, True), _cu(flow_xy, True)
    out = F.BilinearSampler(mx.NDArray(data), F.GridGenerator(mx.NDArray(flow), transform_type="warp"))
    out.backward(mx.NDArray(_cu(go)))
    dr, fr = _cu(img).double().requires_grad_(), _cu(flow_xy).double().requires_grad_()
    ref = _ref_on_cuda(torch_ref.reconstruction2d, dr, fr.flip(1))
    ref.backward(_cu(go).double())
    _close(out.t.detach(), ref.detach())
    _close(data.grad, dr.grad)
    _close(flow.grad, fr.grad)
