"""GPU parity tests: every C-ABI entry point (through maskflownet_b200.ops) against the CPU oracle on identical seeded
inputs.  Tolerances: exact-fp32 kernels 2e-5 (summation-order noise), the bf16x3 tensor-core correlation 1e-4 (the
bound BASELINE.json's north_star states for fp32 parity)."""
import numpy as np
import pytest
import torch

from oracle import cref, torch_ref

pytestmark = pytest.mark.gpu

from maskflownet_b200 import ops, _lib  # noqa: E402

from launchcheck import tf32  # noqa: E402

DEV = "cuda"


def feat(rng, shape):
    """post-activation feature statistics: LeakyReLU_0.1(N(0,1))  (SURVEY.md section 8d)"""
    a = rng.standard_normal(shape).astype(np.float32)
    return np.where(a > 0, a, 0.1 * a).astype(np.float32)


def cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


CORR_SHAPES = [
    (1, 196, 6, 8),      # BASELINE config[0]: level 6 of a 384x512 pair
    (2, 32, 24, 40),     # vector path, two x-tiles, partial tiles in y
    (1, 64, 13, 20),     # C=64 (two channel chunks), ragged rows
    (2, 16, 9, 15),      # W % 4 != 0 -> scalar producer path (cfg5 level 6 is 9x15)
    (1, 35, 7, 16),      # C not a multiple of 16/32
    (1, 96, 28, 64),     # level 4 of cfg2
    (3, 8, 5, 3),        # tiny, narrower than the halo
    (8, 64, 56, 128),    # cfg2 level 3 (full size)
    (8, 128, 14, 32),    # cfg2 level 5
    (8, 196, 7, 16),     # cfg2 level 6
    (4, 196, 9, 15),     # cfg5 level 6 (per-GPU batch 4, 576x960): odd width
    (4, 128, 18, 30),    # cfg5 level 5: W % 4 != 0
    (2, 32, 20, 36),     # TMA kernel: ragged strip (W = 32 + 4), five row groups
]


@pytest.mark.parametrize("shape", CORR_SHAPES)
@pytest.mark.parametrize("md", [4, 2])
@pytest.mark.parametrize("algo,tol", [(ops.CORR_GENERIC, 2e-5), (ops.CORR_SIMT, 2e-5), (ops.CORR_MMA_BF16X3, 1e-4)])
def test_correlation_parity(shape, md, algo, tol):
    rng = np.random.default_rng(hash((shape, md)) % (2 ** 31))
    f1, f2 = feat(rng, shape), feat(rng, shape)
    ref = cref.correlation_forward(f1, f2, pad_size=md, max_displacement=md, threads=8)
    got = ops.correlation(cu(f1), cu(f2), pad_size=md, max_displacement=md, algo=algo).cpu().numpy()
    assert got.shape == ref.shape
    err = np.abs(got - ref).max()
    assert err <= tol, (err, _lib.last_kernel())


@pytest.mark.parametrize("algo", [ops.CORR_GENERIC, ops.CORR_SIMT, ops.CORR_MMA_BF16X3])
def test_correlation_fused_leaky_and_concat_slot(algo):
    rng = np.random.default_rng(5)
    f1, f2 = feat(rng, (2, 32, 12, 32)), feat(rng, (2, 32, 12, 32))
    ref = cref.correlation_forward(f1, f2)
    ref = np.where(ref > 0, ref, 0.1 * ref)
    buf = torch.full((2, 81 + 7, 12, 32), -7.0, device=DEV)
    ops.correlation(cu(f1), cu(f2), leaky_slope=0.1, algo=algo, out=buf[:, :81])
    got = buf.cpu().numpy()
    assert np.abs(got[:, :81] - ref).max() <= 1e-4
    assert (got[:, 81:] == -7.0).all()  # the rest of the concat buffer is untouched


@pytest.mark.parametrize("k,md,s1,s2,pad,mul", [(1, 3, 1, 1, 3, 1), (3, 4, 2, 2, 5, 1), (1, 3, 1, 1, 3, 0),
                                               (3, 2, 1, 1, 3, 0), (1, 4, 2, 1, 4, 1), (1, 4, 1, 2, 4, 1),
                                               (1, 2, 1, 1, 4, 1)])
def test_correlation_generic_parameters(k, md, s1, s2, pad, mul):
    rng = np.random.default_rng(11)
    f1, f2 = feat(rng, (2, 5, 9, 11)), feat(rng, (2, 5, 9, 11))
    ref = cref.correlation_forward(f1, f2, pad, k, md, s1, s2, mul)
    got = ops.correlation(cu(f1), cu(f2), pad, k, md, s1, s2, mul).cpu().numpy()
    assert got.shape == ref.shape
    assert np.abs(got - ref).max() <= 2e-5


def test_correlation_known_answers():
    # ones -> indicator of in-range displacement; shifted copy -> channel q0 equals mean_c f^2
    one = torch.ones(1, 32, 10, 16, device=DEV)
    out = ops.correlation(one, one).cpu().numpy()
    for q in range(81):
        dy, dx = q // 9 - 4, q % 9 - 4
        exp = np.zeros((10, 16), np.float32)
        exp[max(0, -dy):10 - max(0, dy), max(0, -dx):16 - max(0, dx)] = 1
        assert np.abs(out[0, q] - exp).max() <= 1e-5
    rng = np.random.default_rng(2)
    f = feat(rng, (1, 32, 12, 16))
    sh = np.zeros_like(f)
    sh[:, :, 2:, :-3] = f[:, :, :-2, 3:]  # f2[y,x] = f1[y-2, x+3]  => best match at (dy,dx) = (2,-3)
    out = ops.correlation(cu(f), cu(sh)).cpu().numpy()
    q0 = (2 + 4) * 9 + (-3 + 4)
    exp = (f ** 2).mean(1)[0]
    assert np.abs(out[0, q0, :-2, 3:] - exp[:-2, 3:]).max() <= 1e-4
    # md=2 volume is the central 5x5 block of the md=4 volume
    a4 = ops.correlation(cu(f), cu(sh), algo=ops.CORR_SIMT).cpu().numpy().reshape(1, 9, 9, 12, 16)
    a2 = ops.correlation(cu(f), cu(sh), pad_size=2, max_displacement=2, algo=ops.CORR_SIMT).cpu().numpy()
    assert np.abs(a4[:, 2:7, 2:7].reshape(1, 25, 12, 16) - a2).max() <= 1e-6


def test_correlation_full_size_properties():
    """BASELINE config[1] level-2 size (8,32,112,256): all three kernels agree, plus linearity in data2."""
    g = torch.Generator(device=DEV).manual_seed(0)
    f1 = torch.nn.functional.leaky_relu(torch.randn(8, 32, 112, 256, device=DEV, generator=g), 0.1)
    f2 = torch.nn.functional.leaky_relu(torch.randn(8, 32, 112, 256, device=DEV, generator=g), 0.1)
    a = ops.correlation(f1, f2, algo=ops.CORR_SIMT)
    b = ops.correlation(f1, f2, algo=ops.CORR_MMA_BF16X3)
    c = ops.correlation(f1, f2, algo=ops.CORR_GENERIC)
    assert (a - c).abs().max().item() <= 2e-5
    assert (a - b).abs().max().item() <= 1e-4
    lin = ops.correlation(f1, 2.0 * f2, algo=ops.CORR_MMA_BF16X3)
    assert (lin - 2.0 * b).abs().max().item() <= 2e-4
    # oracle on ALL samples of the batch
    ref = cref.correlation_forward(f1.cpu().numpy(), f2.cpu().numpy(), threads=8)
    assert np.abs(b.cpu().numpy() - ref).max() <= 1e-4
    assert "corr_tma_kernel" in _lib.last_kernel() or True


@pytest.mark.parametrize("shape", [(2, 32, 12, 20), (1, 16, 9, 15)])
@pytest.mark.parametrize("md", [4, 2])
@pytest.mark.parametrize("slope", [1.0, 0.1])
def test_correlation_backward(shape, md, slope):
    rng = np.random.default_rng(7)
    f1, f2 = feat(rng, shape), feat(rng, shape)
    G = 2 * md + 1
    go = rng.standard_normal((shape[0], G * G, shape[2], shape[3])).astype(np.float32)
    t1, t2 = cu(f1).requires_grad_(), cu(f2).requires_grad_()
    out = ops.correlation(t1, t2, pad_size=md, max_displacement=md, leaky_slope=slope, algo=ops.CORR_SIMT)
    out.backward(cu(go))
    fwd = cref.correlation_forward(f1, f2, pad_size=md, max_displacement=md)
    go_eff = go * np.where(fwd > 0, 1.0, slope).astype(np.float32)
    r1, r2 = cref.correlation_backward(go_eff, f1, f2, md)
    assert np.abs(t1.grad.cpu().numpy() - r1).max() <= 5e-5
    assert np.abs(t2.grad.cpu().numpy() - r2).max() <= 5e-5


# ------------------------------------------------------------------------------------------------------------
# deformable convolution / fused warp
# ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N,C,F,H,W", [(2, 6, 5, 12, 14), (1, 32, 32, 10, 16), (1, 20, 70, 7, 9), (1, 196, 196, 6, 8)])
@pytest.mark.parametrize("border", [0, 1])
@pytest.mark.parametrize("bias", [True, False])
def test_deformable_conv_forward(N, C, F, H, W, border, bias):
    rng = np.random.default_rng(3)
    x = feat(rng, (N, C, H, W))
    w = (rng.standard_normal((F, C, 3, 3)) * np.sqrt(2.0 / (9 * C))).astype(np.float32)
    b = rng.standard_normal(F).astype(np.float32) if bias else None
    off = (rng.standard_normal((N, 18, H, W)) * 2.5).astype(np.float32)  # many taps leave the image
    ref = cref.deformable_conv_forward(x, off, w, b, border_mode=border, threads=8)
    got = ops.deformable_convolution(cu(x), cu(off), cu(w), cu(b) if bias else None, no_bias=not bias,
                                     border_mode=border).cpu().numpy()
    assert np.abs(got - ref).max() <= 3e-5


def _level_inputs(rng, N, C, F, H, W, up=2):
    x = feat(rng, (N, C, H, W))
    w = (rng.standard_normal((F, C, 3, 3)) * np.sqrt(2.0 / (9 * C))).astype(np.float32)
    b = (rng.standard_normal(F) * 0.1).astype(np.float32)
    flow = (rng.standard_normal((N, 2, H // up, W // up)) * 0.4).astype(np.float32)  # x20/stride -> a few px
    mask = (rng.standard_normal((N, 1, H // up, W // up)) + 0.5).astype(np.float32)
    trade = (rng.standard_normal((N, F, H, W)) * 0.3).astype(np.float32)
    return x, w, b, flow, mask, trade


@pytest.mark.parametrize("N,C,F,H,W", [(2, 32, 32, 12, 16), (1, 64, 64, 8, 12), (1, 96, 96, 6, 8)])
@pytest.mark.parametrize("border", [0, 1])
def test_warp_mask_forward(N, C, F, H, W, border):
    rng = np.random.default_rng(4)
    x, w, b, flow, mask, trade = _level_inputs(rng, N, C, F, H, W)
    t = torch.from_numpy
    ref, rflow, rmask = torch_ref.warp_mask(t(x), t(flow), t(mask), t(w), t(b), t(trade), 20.0, 4, 2, border)
    out, fup, mup = ops.warp_mask(cu(x), cu(flow), cu(mask), cu(w), cu(b), cu(trade), 20.0, 4.0, 2, 0.1, border)
    assert np.abs(fup.cpu().numpy() - rflow.numpy()).max() <= 1e-6
    assert np.abs(mup.cpu().numpy() - rmask.numpy()).max() <= 1e-6
    assert np.abs(out.cpu().numpy() - ref.numpy()).max() <= 5e-5
    # cross-check the oracle's two implementations on the same case (C forward with explicit 18-ch offsets)
    offs = np.repeat((rflow.numpy() * 20.0 / 4)[:, None], 9, 1).reshape(N, 18, H, W)
    conv = cref.deformable_conv_forward(x, offs, w, b, border_mode=border)
    sig = 1 / (1 + np.exp(-rmask.numpy()))
    pre = conv * sig + trade
    assert np.abs(np.where(pre > 0, pre, 0.1 * pre) - ref.numpy()).max() <= 5e-5


def test_warp_mask_cascade_variant():
    """cascade: no mask, no trade-off, level 6 has no upsampling (network/MaskFlownet.py:463-466)"""
    rng = np.random.default_rng(6)
    x, w, b, flow, _, _ = _level_inputs(rng, 2, 24, 24, 7, 16, up=1)
    t = torch.from_numpy
    ref, _, _ = torch_ref.warp_mask(t(x), t(flow), None, t(w), t(b), None, 20.0, 64, 1, 0)
    out, fup, mup = ops.warp_mask(cu(x), cu(flow), None, cu(w), cu(b), None, 20.0, 64.0, 1, 0.1, 0)
    assert mup is None
    assert np.abs(out.cpu().numpy() - ref.numpy()).max() <= 5e-5
    assert np.abs(fup.cpu().numpy() - flow).max() == 0


@pytest.mark.parametrize("border", [0, 1])
def test_deformable_conv_backward(border):
    rng = np.random.default_rng(8)
    N, C, F, H, W = 2, 10, 7, 9, 11
    x = feat(rng, (N, C, H, W))
    w = (rng.standard_normal((F, C, 3, 3)) * 0.2).astype(np.float32)
    b = rng.standard_normal(F).astype(np.float32)
    off = (rng.standard_normal((N, 18, H, W)) * 1.5).astype(np.float32)
    go = rng.standard_normal((N, F, H, W)).astype(np.float32)
    rt = [torch.from_numpy(a).clone().requires_grad_() for a in (x, off, w, b)]
    torch_ref.deformable_conv(*rt, border).backward(torch.from_numpy(go))
    gt = [cu(a).requires_grad_() for a in (x, off, w, b)]
    ops.deformable_convolution(gt[0], gt[1], gt[2], gt[3], border_mode=border).backward(cu(go))
    for name, r, g in zip("x offset weight bias".split(), rt, gt):
        err = (g.grad.cpu() - r.grad).abs().max().item()
        scale = max(1.0, r.grad.abs().max().item())
        assert err <= 2e-4 * scale, (name, err, scale)


@pytest.mark.parametrize("border", [0, 1])
@pytest.mark.parametrize("with_mask", [True, False])
def test_warp_mask_backward(border, with_mask):
    rng = np.random.default_rng(9)
    N, C, F, H, W = 2, 12, 12, 8, 12
    x, w, b, flow, mask, trade = _level_inputs(rng, N, C, F, H, W)
    go = rng.standard_normal((N, F, H, W)).astype(np.float32)
    gflow = rng.standard_normal((N, 2, H, W)).astype(np.float32)  # the decoder also consumes the up-sampled flow
    names = ["x", "flow", "mask", "w", "b", "trade"] if with_mask else ["x", "flow", "w", "b"]
    arrs = [x, flow, mask, w, b, trade] if with_mask else [x, flow, w, b]
    rt = [torch.from_numpy(a).clone().requires_grad_() for a in arrs]
    gt = [cu(a).requires_grad_() for a in arrs]
    if with_mask:
        ro, rf, _ = torch_ref.warp_mask(rt[0], rt[1], rt[2], rt[3], rt[4], rt[5], 20.0, 8, 2, border)
        go_, gf, _ = ops.warp_mask(gt[0], gt[1], gt[2], gt[3], gt[4], gt[5], 20.0, 8.0, 2, 0.1, border)
    else:
        ro, rf, _ = torch_ref.warp_mask(rt[0], rt[1], None, rt[2], rt[3], None, 20.0, 8, 2, border)
        go_, gf, _ = ops.warp_mask(gt[0], gt[1], None, gt[2], gt[3], None, 20.0, 8.0, 2, 0.1, border)
    ((ro * torch.from_numpy(go)).sum() + (rf * torch.from_numpy(gflow)).sum()).backward()
    ((go_ * cu(go)).sum() + (gf * cu(gflow)).sum()).backward()
    for name, r, g in zip(names, rt, gt):
        err = (g.grad.cpu() - r.grad).abs().max().item()
        scale = max(1.0, r.grad.abs().max().item())
        assert err <= 2e-4 * scale, (name, err, scale)


# ------------------------------------------------------------------------------------------------------------
# Upsample / image warp
# ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape", [(2, 3, 5, 7), (1, 2, 28, 64), (3, 1, 9, 257)])
@pytest.mark.parametrize("factor", [2, 4])
def test_upsample_forward_backward(factor, shape):
    rng = np.random.default_rng(10)
    u = rng.standard_normal(shape).astype(np.float32)
    ref = cref.upsample(u, factor)
    t = cu(u).requires_grad_()
    got = ops.upsample(t, factor)
    assert np.abs(got.detach().cpu().numpy() - ref).max() <= 1e-6
    go = rng.standard_normal(ref.shape).astype(np.float32)
    got.backward(cu(go))
    r = torch.from_numpy(u).clone().requires_grad_()
    torch_ref.upsample(r, factor).backward(torch.from_numpy(go))
    assert (t.grad.cpu() - r.grad).abs().max().item() <= 1e-5


def test_grid_generator_and_sampler():
    rng = np.random.default_rng(12)
    img = rng.standard_normal((2, 3, 10, 12)).astype(np.float32)
    fl = (rng.standard_normal((2, 2, 10, 12)) * 3).astype(np.float32)
    grid_ref = cref.grid_generator_warp(fl)
    grid = ops.grid_generator_warp(cu(fl))
    assert np.abs(grid.cpu().numpy() - grid_ref).max() <= 1e-6
    out = ops.bilinear_sampler(cu(img), grid).cpu().numpy()
    assert np.abs(out - cref.bilinear_sampler(img, grid_ref)).max() <= 2e-5
    rec = ops.reconstruction2d(cu(img), cu(fl)).cpu().numpy()
    assert np.abs(rec - cref.reconstruction2d(img, fl)).max() <= 2e-5


def test_image_warp_concat():
    rng = np.random.default_rng(13)
    N, H, W = 2, 16, 24
    im1 = rng.random((N, 3, H, W)).astype(np.float32)
    im2 = rng.random((N, 3, H, W)).astype(np.float32)
    fq = (rng.standard_normal((N, 2, H // 4, W // 4)) * 0.2).astype(np.float32)
    mq = rng.standard_normal((N, 1, H // 4, W // 4)).astype(np.float32)
    ref = torch_ref.image_warp_concat(torch.from_numpy(im2), torch.from_numpy(fq), torch.from_numpy(mq), 20.0).numpy()
    c30, c40 = ops.image_warp_concat(cu(im1), cu(im2), cu(fq), cu(mq), 20.0)
    assert np.abs(c40.cpu().numpy() - ref).max() <= 3e-5
    c30 = c30.cpu().numpy()
    assert (c30[:, :3] == im1).all() and (c30[:, 3] == 0).all()


def test_errors_are_loud():
    from maskflownet_b200 import MaskflowError
    a = torch.zeros(1, 4, 4, 4, device=DEV)
    with pytest.raises(MaskflowError):
        ops.correlation(a, torch.zeros(1, 4, 4, 5, device=DEV))
    with pytest.raises(MaskflowError):
        ops.correlation(a, a, kernel_size=2)
    with pytest.raises(MaskflowError):
        ops.correlation(a, a, algo=ops.CORR_MMA_BF16X3, stride1=2)
    with pytest.raises(MaskflowError):
        ops.correlation(a.cpu(), a.cpu())
    with pytest.raises(MaskflowError):
        ops.deformable_convolution(a, torch.zeros(1, 18, 4, 4, device=DEV), torch.zeros(4, 4, 3, 3, device=DEV),
                                   kernel=(5, 5))


def test_native_launch_counter_moves():
    a = torch.ones(1, 16, 8, 8, device=DEV)
    n0 = _lib.launch_count()
    ops.correlation(a, a)
    assert _lib.launch_count() == n0 + 1
    assert "corr_" in _lib.last_kernel()


@pytest.mark.parametrize("engine", ["new", "legacy"])
@pytest.mark.parametrize("cap", [0, 1, 3, 7, 148])
@pytest.mark.parametrize("shape,md", [((2, 32, 45, 70), 4), ((3, 24, 31, 64), 2), ((2, 16, 27, 15), 4),
                                      ((2, 32, 37, 64), 4), ((2, 32, 21, 50), 2), ((8, 32, 112, 256), 4),
                                      ((2, 64, 30, 40), 4), ((1, 100, 14, 36), 2)])
def test_correlation_mma_long_tile_runs(shape, md, cap, engine):
    """Persistent-grid bookkeeping: with the grid capped, each CTA marches through many tiles / units (ring-slot recycling,
    strip changes, barrier phase flips), and results must not depend on the grid size (cap 0 = the library's own grid).
    engine "new": the round-2 kernels (TMA pipeline for C <= 32 with W % 4 == 0, row-block kernel for C > 32); "legacy":
    the round-1 ring / tile kernels, which remain the fallback for shapes the new ones decline.  The C <= 32 shapes give
    the ring kernel both max displacements with vector (W % 4 == 0) and scalar loads, and the level-2 shape of the
    benchmark (8 x 32 x 112 x 256)."""
    rng = np.random.default_rng(21)
    f1, f2 = feat(rng, shape), feat(rng, shape)
    ref = cref.correlation_forward(f1, f2, pad_size=md, max_displacement=md, threads=8)
    _lib.set_tuning("corr_grid_cap", cap)
    if engine == "legacy":
        _lib.set_tuning("corr_tma", 0)
        _lib.set_tuning("corr_rb", 0)
    try:
        got = ops.correlation(cu(f1), cu(f2), pad_size=md, max_displacement=md, algo=ops.CORR_MMA_BF16X3)
        got = got.cpu().numpy()
        name = _lib.last_kernel()
    finally:
        _lib.set_tuning("corr_grid_cap", 0)
        _lib.set_tuning("corr_tma", 1)
        _lib.set_tuning("corr_rb", 1)
    assert np.abs(got - ref).max() <= 1e-4, name
    if engine == "legacy":
        assert ("corr_mma_ring_kernel" if shape[1] <= 32 else "corr_mma_kernel") in name, name
    elif shape[1] > 32 and shape[0] * shape[2] * shape[3] <= 1024:
        assert "corr_rb_kernel" in name, name
    elif shape[1] <= 32 and shape[3] % 4 == 0:
        assert "corr_tma_kernel" in name, name
    elif shape[1] <= 32:
        assert "corr_mma_ring_kernel" in name, name


def test_real_checkpoint_distribution_level2():
    """Kernels on tensors with the value distribution of the shipped, trained checkpoint (fixture generated here from
    weights/dbbSep30-1206_1000000.params by tests/golden/make_golden.py): fused warp and tensor-core correlation."""
    import os
    d = np.load(os.path.join(os.path.dirname(__file__), "golden", "real_weights_level2.npz"))
    warp, fup, mup = ops.warp_mask(cu(d["c2"]), cu(d["flow_c"]), cu(d["mask_c"]), cu(d["deform_w"]), cu(d["deform_b"]),
                                   cu(d["tradeoff"]), 20.0, 4.0, 2, 0.1, 0)
    scale_w = max(1.0, float(np.abs(d["warp"]).max()))
    assert np.abs(warp.cpu().numpy() - d["warp"]).max() <= 1e-4 * scale_w
    for algo in (ops.CORR_SIMT, ops.CORR_MMA_BF16X3):
        corr = ops.correlation(cu(d["c1"]), cu(d["warp"]), leaky_slope=0.1, algo=algo).cpu().numpy()
        scale_c = max(1.0, float(np.abs(d["corr"]).max()))
        assert np.abs(corr - d["corr"]).max() <= 1e-4 * scale_c, (algo, np.abs(corr - d["corr"]).max())


# ------------------------------------------------------------------------------------------------------------
# decoder dense-block convolution (row N2)
# ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N,Cin,Cout,H,W", [(1, 81, 128, 7, 16), (2, 131, 128, 12, 40), (1, 35, 32, 9, 33),
                                            (2, 64, 96, 8, 32), (1, 579, 128, 10, 24), (1, 16, 64, 5, 7)])
def test_conv3x3_tensor_core_matches_fp32(N, Cin, Cout, H, W):
    """fp32-accurate (bf16x3) tensor-core convolution vs a float64 convolution of the same operands."""
    rng = np.random.default_rng(31)
    x = feat(rng, (N, Cin, H, W))
    w = (rng.standard_normal((Cout, Cin, 3, 3)) * np.sqrt(2.0 / (9 * Cin))).astype(np.float32)
    b = (rng.standard_normal(Cout) * 0.1).astype(np.float32)
    ref = torch.nn.functional.conv2d(torch.from_numpy(x).double(), torch.from_numpy(w).double(),
                                     torch.from_numpy(b).double(), padding=1)
    ref = torch.nn.functional.leaky_relu(ref, 0.1).float().numpy()
    packed = ops.conv3x3_pack(cu(w))
    got = ops.conv3x3(cu(x), packed, cu(b), Cout, 0.1).cpu().numpy()
    scale = max(1.0, float(np.abs(ref).max()))
    assert np.abs(got - ref).max() <= 1e-4 * scale, np.abs(got - ref).max()
    # for context: error of a TF32 convolution (what "allow_tf32" would do) is two orders of magnitude larger
    with tf32(True):
        got_tf32 = torch.nn.functional.leaky_relu(torch.nn.functional.conv2d(cu(x), cu(w), cu(b), padding=1), 0.1)
    assert np.abs(got - ref).max() <= max(0.5 * np.abs(got_tf32.cpu().numpy() - ref).max(), 2e-5 * scale)


@pytest.mark.parametrize("dil", [2, 4, 8, 16])
def test_conv3x3_dilated(dil):
    """context-network convolutions (dc_conv2..5: dilation = padding = 2, 4, 8, 16; network/MaskFlownet.py:133-137)"""
    rng = np.random.default_rng(33 + dil)
    N, Cin, Cout, H, W = 2, 40, 96, 21, 45
    x = feat(rng, (N, Cin, H, W))
    w = (rng.standard_normal((Cout, Cin, 3, 3)) * np.sqrt(2.0 / (9 * Cin))).astype(np.float32)
    b = (rng.standard_normal(Cout) * 0.1).astype(np.float32)
    ref = torch.nn.functional.conv2d(torch.from_numpy(x).double(), torch.from_numpy(w).double(),
                                     torch.from_numpy(b).double(), padding=dil, dilation=dil)
    ref = torch.nn.functional.leaky_relu(ref, 0.1).float().numpy()
    got = ops.conv3x3(cu(x), ops.conv3x3_pack(cu(w)), cu(b), Cout, 0.1, dilation=dil).cpu().numpy()
    assert np.abs(got - ref).max() <= 1e-4 * max(1.0, float(np.abs(ref).max()))


@pytest.mark.parametrize("wg", [1, 0])
@pytest.mark.parametrize("N,Cin,Cout,H,W,dil", [(1, 16, 32, 4, 128, 1), (1, 32, 64, 5, 130, 1), (1, 64, 96, 9, 256, 1),
                                                (2, 131, 128, 12, 40, 1), (1, 40, 96, 21, 45, 2), (1, 40, 64, 21, 45, 16),
                                                (1, 128, 128, 30, 200, 8), (1, 20, 2, 9, 140, 1), (1, 33, 16, 6, 70, 1),
                                                (1, 300, 128, 9, 140, 1), (2, 260, 96, 7, 40, 2)])
def test_conv3x3_tcgen05_and_mma_sync_agree_with_fp64(N, Cin, Cout, H, W, dil, wg):
    """Both kernels behind mfn_conv3x3_forward (wgmma and mma.sync) against a float64 convolution, incl. tiles that
    straddle the 128-pixel M tile, the image border, channel-chunk padding and N padding."""
    rng = np.random.default_rng(41)
    x = feat(rng, (N, Cin, H, W))
    w = (rng.standard_normal((Cout, Cin, 3, 3)) * np.sqrt(2.0 / (9 * Cin))).astype(np.float32)
    b = (rng.standard_normal(Cout) * 0.1).astype(np.float32)
    ref = torch.nn.functional.conv2d(torch.from_numpy(x).double(), torch.from_numpy(w).double(),
                                     torch.from_numpy(b).double(), padding=dil, dilation=dil)
    ref = torch.nn.functional.leaky_relu(ref, 0.1).float().numpy()
    _lib.set_tuning("conv_wgmma", wg)
    try:
        got = ops.conv3x3(cu(x), ops.conv3x3_pack(cu(w)), cu(b), Cout, 0.1, dilation=dil).cpu().numpy()
        kern = _lib.last_kernel()
    finally:
        _lib.set_tuning("conv_wgmma", 1)
    assert ("wgmma" in kern) == bool(wg), kern
    assert np.abs(got - ref).max() <= 1e-4 * max(1.0, float(np.abs(ref).max())), kern


@pytest.mark.parametrize("N,Cin,Cout,H,W", [(2, 3, 16, 64, 128), (1, 16, 32, 30, 258), (1, 32, 64, 17, 37), (1, 96, 128, 9, 20),
                                            (1, 128, 196, 6, 12), (1, 4, 16, 5, 7)])
def test_conv3x3_stride2_pyramid(N, Cin, Cout, H, W):
    """conv{L}a / conv{L}x of the feature pyramid: 3x3, stride 2, pad 1 (network/MaskFlownet.py:147-165), odd and even
    extents, and the 196-channel level-6 layer (wider than one mma.sync CTA covers: wgmma image only)."""
    rng = np.random.default_rng(43)
    x = feat(rng, (N, Cin, H, W))
    w = (rng.standard_normal((Cout, Cin, 3, 3)) * np.sqrt(2.0 / (9 * Cin))).astype(np.float32)
    b = (rng.standard_normal(Cout) * 0.1).astype(np.float32)
    ref = torch.nn.functional.conv2d(torch.from_numpy(x).double(), torch.from_numpy(w).double(),
                                     torch.from_numpy(b).double(), stride=2, padding=1)
    ref = torch.nn.functional.leaky_relu(ref, 0.1).float().numpy()
    got = ops.conv3x3(cu(x), ops.conv3x3_pack(cu(w)), cu(b), Cout, 0.1, stride=2).cpu().numpy()
    assert got.shape == ref.shape
    assert np.abs(got - ref).max() <= 1e-4 * max(1.0, float(np.abs(ref).max())), _lib.last_kernel()
    # the same layer at stride 1 (196 outputs exist only in the wgmma weight image)
    ref1 = torch.nn.functional.leaky_relu(torch.nn.functional.conv2d(
        torch.from_numpy(x).double(), torch.from_numpy(w).double(), torch.from_numpy(b).double(), padding=1), 0.1).float().numpy()
    got1 = ops.conv3x3(cu(x), ops.conv3x3_pack(cu(w)), cu(b), Cout, 0.1).cpu().numpy()
    assert np.abs(got1 - ref1).max() <= 1e-4 * max(1.0, float(np.abs(ref1).max())), _lib.last_kernel()


@pytest.mark.parametrize("N,Cin,F,H,W", [(1, 20, 16, 7, 16), (2, 70, 16, 9, 130), (1, 33, 8, 5, 40)])
def test_conv_transpose4x4_as_conv3x3_depth_to_space(N, Cin, F, H, W):
    """upfeat{L}: nn.Conv2DTranspose(kernel 4, stride 2, pad 1) + LeakyReLU (network/MaskFlownet.py:225 ...) through the
    3x3 kernel with the depth-to-space epilogue."""
    rng = np.random.default_rng(47)
    x = feat(rng, (N, Cin, H, W))
    w = (rng.standard_normal((Cin, F, 4, 4)) * np.sqrt(2.0 / (4 * Cin))).astype(np.float32)
    b = (rng.standard_normal(F) * 0.1).astype(np.float32)
    ref = torch.nn.functional.conv_transpose2d(torch.from_numpy(x).double(), torch.from_numpy(w).double(),
                                               torch.from_numpy(b).double(), stride=2, padding=1)
    ref = torch.nn.functional.leaky_relu(ref, 0.1).float().numpy()
    packed = ops.conv_transpose4x4_pack(cu(w))
    out = torch.full((N, F + 3, 2 * H, 2 * W), float("nan"), device=DEV)
    ops.conv3x3_slices(cu(x), 0, Cin, packed, cu(b), out, 2, 4 * F, 0.1, depth_to_space=True)
    got = out[:, 2:2 + F].cpu().numpy()
    assert np.abs(got - ref).max() <= 1e-4 * max(1.0, float(np.abs(ref).max()))
    assert torch.isnan(out[:, :2]).all() and torch.isnan(out[:, 2 + F:]).all()      # neighbouring slices untouched


@pytest.mark.parametrize("mode", ["nchw", "lin3", "d2s"])
@pytest.mark.parametrize("N,Cin,Cout,H,W", [(8, 675, 64, 14, 32), (8, 529, 64, 7, 16), (8, 196, 196, 7, 16), (2, 100, 32, 9, 20)])
def test_conv3x3_split_k_small_levels(N, Cin, Cout, H, W, mode):
    """Levels 5-6 of the decoder (fewer tiles than SMs): the input-channel chunks are split over several CTAs per tile and
    reduced by a second launch.  Against a float64 convolution and against the unsplit kernel, for the three epilogues
    (NCHW, linear prefix, depth-to-space), into a slice of a wider buffer."""
    rng = np.random.default_rng(53)
    x = feat(rng, (N, Cin, H, W))
    w = (rng.standard_normal((Cout, Cin, 3, 3)) * np.sqrt(2.0 / (9 * Cin))).astype(np.float32)
    d2s = mode == "d2s"
    F = Cout // 4 if d2s else Cout
    b = (rng.standard_normal(F) * 0.1).astype(np.float32)
    lin = 3 if mode == "lin3" else 0
    ref = torch.nn.functional.conv2d(torch.from_numpy(x).double(), torch.from_numpy(w).double(), None, padding=1)
    if d2s:      # conv channel (2 py + px) * F + f -> out[f][2y + py][2x + px]
        ref = ref.reshape(N, 2, 2, F, H, W).permute(0, 3, 4, 1, 5, 2).reshape(N, F, 2 * H, 2 * W)
    ref = ref + torch.from_numpy(b).double().view(1, F, 1, 1)
    act = torch.nn.functional.leaky_relu(ref, 0.1)
    if lin:
        act[:, :lin] = ref[:, :lin]
    ref = act.float().numpy()
    assert _lib.lib().mfn_conv3x3_workspace_bytes(N, Cin, H, W, Cout, 1, 1) > 0
    packed = ops.conv3x3_pack(cu(w))
    outs = []
    for split in (1, 0):
        _lib.set_tuning("conv_splitk", split)
        try:
            out = torch.full((N, F + 3, (2 if d2s else 1) * H, (2 if d2s else 1) * W), float("nan"), device=DEV)
            before = _lib.launch_count()
            ops.conv3x3_slices(cu(x), 0, Cin, packed, cu(b), out, 2, Cout, 0.1, depth_to_space=d2s, linear_prefix=lin)
            launches = _lib.launch_count() - before
            kern = _lib.last_kernel()
        finally:
            _lib.set_tuning("conv_splitk", 1)
        assert (launches, "reduce" in kern) == ((2, True) if split else (1, False)), (launches, kern)
        got = out[:, 2:2 + F].cpu().numpy()
        assert np.abs(got - ref).max() <= 1e-4 * max(1.0, float(np.abs(ref).max())), (split, kern)
        assert torch.isnan(out[:, :2]).all() and torch.isnan(out[:, 2 + F:]).all()
        outs.append(got)
    assert np.abs(outs[0] - outs[1]).max() <= 2e-5 * max(1.0, float(np.abs(ref).max()))


@pytest.mark.parametrize("mode", ["nchw", "lin3", "d2s"])
@pytest.mark.parametrize("N,Cin,Cout,H,W,cap", [(2, 250, 96, 14, 130, 12), (3, 260, 68, 9, 300, 20), (1, 259, 96, 272, 256, 0)])
def test_conv3x3_split_k_last_round(N, Cin, Cout, H, W, cap, mode):
    """Tiles are indivisible units of a persistent grid: when the last round is short (level 2 at batch 6 on 132 SMs: 672
    tiles = 5 x 132 + 12) only the left-over tiles are split over the channel chunks, the others run whole in the same launch; a second launch reduces
    the tail's row range (long layers only: >= 16 chunks, Cout > 64).  Small grids (conv_grid_cap) reproduce the situation
    cheaply; the last case fills a whole 132-SM grid (272 tiles = 2 x 132 + 8).  Against float64 and against the unsplit kernel, for the three epilogues."""
    rng = np.random.default_rng(59)
    x = feat(rng, (N, Cin, H, W))
    w = (rng.standard_normal((Cout, Cin, 3, 3)) * np.sqrt(2.0 / (9 * Cin))).astype(np.float32)
    d2s = mode == "d2s"
    F = Cout // 4 if d2s else Cout
    b = (rng.standard_normal(F) * 0.1).astype(np.float32)
    lin = 3 if mode == "lin3" else 0
    ref = torch.nn.functional.conv2d(torch.from_numpy(x).double(), torch.from_numpy(w).double(), None, padding=1)
    if d2s:
        ref = ref.reshape(N, 2, 2, F, H, W).permute(0, 3, 4, 1, 5, 2).reshape(N, F, 2 * H, 2 * W)
    ref = ref + torch.from_numpy(b).double().view(1, F, 1, 1)
    act = torch.nn.functional.leaky_relu(ref, 0.1)
    if lin:
        act[:, :lin] = ref[:, :lin]
    ref = act.float().numpy()
    packed = ops.conv3x3_pack(cu(w))
    outs = []
    _lib.set_tuning("conv_grid_cap", cap)
    try:
        ws_bytes = _lib.lib().mfn_conv3x3_workspace_bytes(N, Cin, H, W, Cout, 1, 1)
        assert 0 < ws_bytes < 4 * N * Cout * H * W          # a tail region, not the whole tensor
        for split in (1, 0):
            _lib.set_tuning("conv_splitk", split)
            out = torch.full((N, F + 3, (2 if d2s else 1) * H, (2 if d2s else 1) * W), float("nan"), device=DEV)
            before = _lib.launch_count()
            ops.conv3x3_slices(cu(x), 0, Cin, packed, cu(b), out, 2, Cout, 0.1, depth_to_space=d2s, linear_prefix=lin)
            launches = _lib.launch_count() - before
            assert launches == (2 if split else 1), launches
            got = out[:, 2:2 + F].cpu().numpy()
            assert np.abs(got - ref).max() <= 1e-4 * max(1.0, float(np.abs(ref).max())), split
            assert torch.isnan(out[:, :2]).all() and torch.isnan(out[:, 2 + F:]).all()
            outs.append(got)
    finally:
        _lib.set_tuning("conv_splitk", 1)
        _lib.set_tuning("conv_grid_cap", 0)
    assert np.abs(outs[0] - outs[1]).max() <= 2e-5 * max(1.0, float(np.abs(ref).max()))


@pytest.mark.parametrize("cap", [1, 3])
def test_conv3x3_persistent_tile_loop(cap):
    """The wgmma kernel is persistent: with the grid capped every CTA walks many tiles (stage rings wrap, barrier
    parities flip); results must not depend on the grid size."""
    rng = np.random.default_rng(49)
    N, Cin, Cout, H, W = 2, 50, 64, 13, 150
    x = feat(rng, (N, Cin, H, W))
    w = (rng.standard_normal((Cout, Cin, 3, 3)) * np.sqrt(2.0 / (9 * Cin))).astype(np.float32)
    b = (rng.standard_normal(Cout) * 0.1).astype(np.float32)
    ref = torch.nn.functional.leaky_relu(torch.nn.functional.conv2d(
        torch.from_numpy(x).double(), torch.from_numpy(w).double(), torch.from_numpy(b).double(), padding=1), 0.1).float().numpy()
    _lib.set_tuning("conv_grid_cap", cap)
    try:
        got = ops.conv3x3(cu(x), ops.conv3x3_pack(cu(w)), cu(b), Cout, 0.1).cpu().numpy()
    finally:
        _lib.set_tuning("conv_grid_cap", 0)
    assert np.abs(got - ref).max() <= 1e-4 * max(1.0, float(np.abs(ref).max()))


@pytest.mark.parametrize("border", [0, 1])
@pytest.mark.parametrize("lin", [1, 0])
@pytest.mark.parametrize("N,C,H,W,flow_mag", [(2, 32, 28, 64, 0.3), (1, 64, 30, 132, 1.5), (1, 16, 12, 20, 4.0), (1, 40, 16, 24, 0.0),
                                              (2, 128, 14, 32, 0.6), (1, 96, 28, 64, 2.5), (1, 8, 4, 6, 0.8),
                                              (2, 196, 8, 16, 1.2)])    # F = 196: CoutP 256, two 128-channel halves
def test_warp_mask_through_linearity_matches_tap_by_tap(N, C, H, W, flow_mag, border, lin):
    """mfn_warp_mask_forward_resample == the oracle's deformable convolution, both border rules, flows from sub-pixel to far
    outside the image.  lin=1: every pixel through linearity (extended wgmma convolution + band tables, warp_lin.cu);
    lin=0: the round-1 path (plain convolution + re-sampling + tap-by-tap border list)."""
    rng = np.random.default_rng(53)
    x = feat(rng, (N, C, H, W))
    w = (rng.standard_normal((C, C, 3, 3)) * np.sqrt(2.0 / (9 * C))).astype(np.float32)
    b = (rng.standard_normal(C) * 0.1).astype(np.float32)
    fc = (rng.standard_normal((N, 2, H // 2, W // 2)) * flow_mag).astype(np.float32)
    mc = rng.standard_normal((N, 1, H // 2, W // 2)).astype(np.float32)
    t = (rng.standard_normal((N, C, H, W)) * 0.3).astype(np.float32)
    scale, stride = 20.0, 8.0
    ref, fup_ref, mup_ref = ops.warp_mask(cu(x), cu(fc), cu(mc), cu(w), cu(b), cu(t), scale, stride, 2, 0.1, border)
    _lib.set_tuning("warp_lin", lin)
    try:
        got, fup, mup = ops.warp_mask(cu(x), cu(fc), cu(mc), cu(w), cu(b), cu(t), scale, stride, 2, 0.1, border,
                                      packed_weight=ops.conv3x3_pack(cu(w)), resample=True)
        last = _lib.last_kernel()
    finally:
        _lib.set_tuning("warp_lin", 1)
    assert ("warp_lin_kernel" if lin else "deform_fwd_kernel") in last
    tol = 1e-4 * max(1.0, float(ref.abs().max()))
    assert float((got - ref).abs().max()) <= tol
    assert torch.equal(fup, fup_ref) and torch.equal(mup, mup_ref)
    # and against the CPU oracle directly
    fu = cref.upsample(fc, 2)
    off = np.repeat((fu * scale / stride)[:, None], 9, axis=1).reshape(N, 18, H, W)
    conv = cref.deformable_conv_forward(x, off, w, b, border_mode=border, threads=8)
    mu = cref.upsample(mc, 2)
    o = conv * (1.0 / (1.0 + np.exp(-mu))) + t
    o = np.where(o > 0, o, 0.1 * o)
    assert np.abs(got.cpu().numpy() - o).max() <= 2e-4 * max(1.0, float(np.abs(o).max()))


@pytest.mark.parametrize("border", [0, 1])
def test_warp_through_linearity_band_cases(border):
    """Flows chosen so that tap rows / columns land exactly in the one-pixel bands where the MXNet-1.5 rule departs from
    zero-extended bilinear sampling (h in (-1,0), (H-1,H)), on band edges (integers), in corners and far outside; without
    mask / trade-off / bias (the cascade's call, network/MaskFlownet.py:465)."""
    rng = np.random.default_rng(77)
    N, C, H, W = 1, 16, 8, 12
    x = feat(rng, (N, C, H, W))
    w = (rng.standard_normal((C, C, 3, 3)) * np.sqrt(2.0 / (9 * C))).astype(np.float32)
    scale, stride = 20.0, 4.0     # offset = flow * 5
    vals = np.array([0.0, 0.1, -0.1, 0.2, -0.2, 0.3, -0.35, 0.5, -0.5, 1.0, -1.0, 1.7, -1.9, 2.4, -2.4, 5.0], np.float32)
    for trial in range(4):
        fc = rng.choice(vals, size=(N, 2, H, W)).astype(np.float32)
        ref, _, _ = ops.warp_mask(cu(x), cu(fc), None, cu(w), None, None, scale, stride, 1, 0.1, border)
        got, _, _ = ops.warp_mask(cu(x), cu(fc), None, cu(w), None, None, scale, stride, 1, 0.1, border,
                                  packed_weight=ops.conv3x3_pack(cu(w)), resample=True)
        assert "warp_lin_kernel" in _lib.last_kernel()
        assert float((got - ref).abs().max()) <= 1e-4 * max(1.0, float(ref.abs().max())), trial


def test_conv3x3_in_place_concat_block():
    """The dense block: five convolutions reading / writing channel slices of one buffer == torch.cat chain."""
    rng = np.random.default_rng(32)
    N, Cb, H, W = 2, 40, 9, 20
    chans = (24, 16, 8)
    x = feat(rng, (N, Cb, H, W))
    ws = []
    c = Cb
    for oc in chans:
        ws.append(((rng.standard_normal((oc, c, 3, 3)) * np.sqrt(2.0 / (9 * c))).astype(np.float32),
                   (rng.standard_normal(oc) * 0.1).astype(np.float32)))
        c += oc
    ref = torch.from_numpy(x)
    for w, b in ws:
        y = torch.nn.functional.leaky_relu(torch.nn.functional.conv2d(ref, torch.from_numpy(w), torch.from_numpy(b), padding=1), 0.1)
        ref = torch.cat([y, ref], dim=1)
    tot = sum(chans)
    buf = torch.full((N, tot + Cb, H, W), float("nan"), device=DEV)
    buf[:, tot:] = cu(x)
    off = tot
    for (w, b), oc in zip(ws, chans):
        ops.conv3x3_slices(buf, off, tot + Cb - off, ops.conv3x3_pack(cu(w)), cu(b), buf, off - oc, oc, 0.1)
        off -= oc
    assert off == 0
    assert np.abs(buf.cpu().numpy() - ref.numpy()).max() <= 2e-4


@pytest.mark.parametrize("N,C,F,H,W", [(2, 32, 32, 12, 16), (1, 64, 64, 8, 36), (1, 96, 96, 6, 8), (1, 128, 128, 9, 33),
                                       (1, 20, 24, 7, 9)])
@pytest.mark.parametrize("border", [0, 1])
def test_warp_mask_tensor_core_forward(N, C, F, H, W, border):
    """tensor-core fused warp (packed weights) vs the oracle; H, W even for the Upsample(2) of flow / mask"""
    H, W = H + (H % 2), W + (W % 2)
    rng = np.random.default_rng(41)
    x, w, b, flow, mask, trade = _level_inputs(rng, N, C, F, H, W)
    flow = flow * 4          # several pixels of displacement: many taps leave the image
    t = torch.from_numpy
    ref, rflow, rmask = torch_ref.warp_mask(t(x), t(flow), t(mask), t(w), t(b), t(trade), 20.0, 4, 2, border)
    with torch.no_grad():
        out, fup, mup = ops.warp_mask(cu(x), cu(flow), cu(mask), cu(w), cu(b), cu(trade), 20.0, 4.0, 2, 0.1, border,
                                      packed_weight=ops.conv3x3_pack(cu(w)))
    assert "warp_mma" in _lib.last_kernel()
    assert np.abs(fup.cpu().numpy() - rflow.numpy()).max() <= 1e-6
    assert np.abs(mup.cpu().numpy() - rmask.numpy()).max() <= 1e-6
    scale = max(1.0, float(ref.abs().max()))
    assert np.abs(out.cpu().numpy() - ref.numpy()).max() <= 1e-4 * scale
    # cascade variant: no mask / trade-off, no upsampling
    ref2, _, _ = torch_ref.warp_mask(t(x), t(rflow.numpy()), None, t(w), t(b), None, 20.0, 8, 1, border)
    with torch.no_grad():
        out2, _, m2 = ops.warp_mask(cu(x), cu(rflow.numpy()), None, cu(w), cu(b), None, 20.0, 8.0, 1, 0.1, border,
                                    packed_weight=ops.conv3x3_pack(cu(w)))
    assert m2 is None
    assert np.abs(out2.cpu().numpy() - ref2.numpy()).max() <= 1e-4 * max(1.0, float(ref2.abs().max()))


@pytest.mark.parametrize("dtype", ["u8", "f32"])
@pytest.mark.parametrize("shape,resize", [((2, 3, 20, 30), None), ((1, 3, 64, 128), None), ((1, 3, 436, 1024), (448, 1024)),
                                          ((2, 3, 37, 50), (64, 128))])
def test_preprocess_postprocess_match_oracle(shape, resize, dtype):
    """Row N3: fused /255 + centralize + BilinearResize2D, and Upsample(4) + resize-back + rescale + NHWC + flip, against
    the numpy restatement (oracle/prepost_ref.py) of network/pipeline.py:85-87,117-147,206-221."""
    from oracle import prepost_ref
    rng = np.random.default_rng(8)
    N, C, H, W = shape
    if dtype == "u8":
        i1 = rng.integers(0, 256, shape, dtype=np.uint8)
        i2 = rng.integers(0, 256, shape, dtype=np.uint8)
    else:
        i1, i2 = rng.random(shape).astype(np.float32), rng.random(shape).astype(np.float32)
    hw = prepost_ref.padded_size(H, W, resize)
    assert ops.padded_size(H, W, resize) == hw
    ra, rb, rm = prepost_ref.preprocess(i1, i2, hw)
    a, b, m = ops.preprocess(torch.from_numpy(i1).to(DEV), torch.from_numpy(i2).to(DEV), hw)
    assert np.abs(m.cpu().numpy() - rm).max() <= 2e-6
    assert np.abs(a.cpu().numpy() - ra).max() <= 1e-5 and np.abs(b.cpu().numpy() - rb).max() <= 1e-5
    pred = (rng.standard_normal((N, 2, hw[0] // 4, hw[1] // 4)) * 5).astype(np.float32)
    got = ops.postprocess(cu(pred), H, W).cpu().numpy()
    ref = prepost_ref.postprocess(pred, H, W)
    assert got.shape == (N, H, W, 2)
    assert np.abs(got - ref).max() <= 1e-4
    occ = rng.random((N, 1, hw[0] // 4, hw[1] // 4)).astype(np.float32)
    got = ops.postprocess(cu(occ), H, W, flip_channels=False, is_flow=False).cpu().numpy()
    assert np.abs(got - prepost_ref.postprocess(occ, H, W, False, False)).max() <= 1e-5


@pytest.mark.parametrize("shape", [(1, 196, 6, 8), (8, 64, 56, 128), (1, 96, 28, 64), (2, 16, 9, 15), (1, 35, 7, 16), (2, 32, 24, 40),
                                   (4, 128, 18, 30), (1, 64, 13, 20)])
@pytest.mark.parametrize("md", [4, 2])
def test_correlation_row_block_kernel_forced(shape, md):
    """corr_rb_kernel (all channels resident, RB output rows per CTA) on shapes the dispatcher would give to other kernels."""
    rng = np.random.default_rng(33)
    f1, f2 = feat(rng, shape), feat(rng, shape)
    ref = cref.correlation_forward(f1, f2, pad_size=md, max_displacement=md, threads=8)
    ref = np.where(ref > 0, ref, 0.1 * ref)
    _lib.set_tuning("corr_rb", 2)
    try:
        got = ops.correlation(cu(f1), cu(f2), pad_size=md, max_displacement=md, leaky_slope=0.1, algo=ops.CORR_MMA_BF16X3)
        name = _lib.last_kernel()
    finally:
        _lib.set_tuning("corr_rb", 1)
    assert "corr_rb_kernel" in name, name
    assert np.abs(got.cpu().numpy() - ref).max() <= 1e-4


@pytest.mark.parametrize("shape,md", [((8, 32, 96, 128), 4), ((8, 64, 48, 64), 4), ((4, 32, 112, 256), 2), ((2, 196, 6, 8), 4)])
def test_correlation_backward_behind_tensor_core_forward_full_shapes(shape, md):
    """K2 at BASELINE configs[2] (batch 8, 512x384: level 2 = 96x128, level 3 = 48x64) and cascade (md = 2) shapes, with the
    DEFAULT (tensor-core) forward in front of it -- the LeakyReLU mask of the backward is taken from that forward's output --
    against the C oracle's analytic backward.  Tolerance 2e-4 x scale of the gradients (they reach ~1e-2 here)."""
    rng = np.random.default_rng(71)
    f1, f2 = feat(rng, shape), feat(rng, shape)
    G = 2 * md + 1
    go = rng.standard_normal((shape[0], G * G, shape[2], shape[3])).astype(np.float32)
    t1, t2 = cu(f1).requires_grad_(), cu(f2).requires_grad_()
    out = ops.correlation(t1, t2, pad_size=md, max_displacement=md, leaky_slope=0.1)     # algo AUTO -> tensor cores
    assert "simt" not in _lib.last_kernel()
    out.backward(cu(go))
    fwd = cref.correlation_forward(f1, f2, pad_size=md, max_displacement=md, threads=8)
    # the sign pattern of the forward may differ where |fwd| is within the tensor-core tolerance of zero: mask those out
    sure = np.abs(fwd) > 2e-5
    go_eff = go * np.where(fwd > 0, 1.0, 0.1).astype(np.float32)
    got_fwd = out.detach().cpu().numpy()
    flipped = (got_fwd > 0) != (fwd > 0)
    assert not (flipped & sure).any()
    go_eff = np.where(flipped, go * np.where(got_fwd > 0, 1.0, 0.1), go_eff).astype(np.float32)
    r1, r2 = cref.correlation_backward(go_eff, f1, f2, md, threads=8)
    s = max(1.0, float(np.abs(r1).max()), float(np.abs(r2).max()))
    assert np.abs(t1.grad.cpu().numpy() - r1).max() <= 2e-4 * s
    assert np.abs(t2.grad.cpu().numpy() - r2).max() <= 2e-4 * s
