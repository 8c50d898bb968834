"""Deterministic mode: the *_det entry points (csrc/det.cuh, det_bwd.cu and the DET kernels of warp_bwd.cu,
image_warp_bwd.cu, prepost.cu), their selection by torch.use_deterministic_algorithms in ops, and
PipelineFlownet(deterministic=True).

CPU: the fixed-point scatter and the ordered reductions compiled for the host (tests/host_emu/det_emu.cpp), run with the
threads in shuffled orders: bit-identical results, within the documented bound of a float64 sum, no overflow when every
sample lands on one pixel, NaN for NaN / inf gradients; the workspace checks of the five entry points.
GPU: every *_det entry against oracle/torch_ref.py and against the atomic path, bit-identical on repeated calls; the op
layer calls exactly the old entry points with the flag off; two fresh processes train to bit-identical parameters.
"""
import contextlib
import ctypes
import json
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

from maskflownet_b200 import _lib, ops
from oracle import torch_ref

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


@contextlib.contextmanager
def det_mode(on=True, warn_only=False):
    """torch.use_deterministic_algorithms(on) inside the block; the previous setting is restored afterwards"""
    prev, prev_warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(on, warn_only=warn_only)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(prev, warn_only=prev_warn)


def _ptr(a):
    return None if a is None else a.ctypes.data_as(ctypes.c_void_p)


# ---------------------------------------------------------------------------------------------------------------
# CPU: the kernel source on the host
# ---------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("emu") / "libdet_emu.so")
    src = os.path.join(HERE, "host_emu", "det_emu.cpp")
    subprocess.run(["g++", "-O1", "-ffp-contract=off", "-shared", "-fPIC", "-I", os.path.join(HERE, "host_emu"), "-o", out, src],
                   check=True)
    L = ctypes.CDLL(out)
    L.emu_det_bits.argtypes = [ctypes.c_longlong]
    L.emu_det_scale.argtypes = [ctypes.c_float, ctypes.c_float, ctypes.c_int, ctypes.c_int, ctypes.POINTER(ctypes.c_int)]
    L.emu_bilinear_sampler_backward_det.argtypes = [ctypes.c_void_p] * 5 + [ctypes.c_int] * 6 + [ctypes.c_void_p]
    L.emu_pixel_abs_sum_max.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_longlong]
    L.emu_pixel_abs_sum_max.restype = ctypes.c_float
    L.emu_ordered_sum.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_longlong, ctypes.c_longlong, ctypes.c_void_p,
                                  ctypes.c_longlong, ctypes.c_int, ctypes.c_void_p]
    return L


def _scale_exp(emu, bound, fanin):
    fin = ctypes.c_int()
    s = emu.emu_det_scale(float(bound), 1.0, 1, emu.emu_det_bits(fanin), ctypes.byref(fin))
    return s, bool(fin.value)


def _sampler_contributions(go, grid, H, W):
    """the fp32 contributions grad_out * corner weight of the sampler backward, computed with the kernel's fp32 operations
    (sampling.cuh), and their float64 sum per data element plus the number of contributions each element receives"""
    N, C, OH, OW = go.shape
    f = np.float32
    gx, gy = grid[:, 0], grid[:, 1]
    xr = (gx + f(1)) * f(W - 1) / f(2)
    yr = (gy + f(1)) * f(H - 1) / f(2)
    x0, y0 = np.floor(xr), np.floor(yr)
    wx0, wy0 = f(1) - (xr - x0), f(1) - (yr - y0)
    wx1, wy1 = f(1) - wx0, f(1) - wy0
    x0, y0 = x0.astype(np.int64), y0.astype(np.int64)
    ref = np.zeros((N, C, H, W), np.float64)
    count = np.zeros((N, C, H, W), np.int64)
    n_idx = np.arange(N)[:, None, None]
    for dy, dx, w in ((0, 0, wy0 * wx0), (0, 1, wy0 * wx1), (1, 0, wy1 * wx0), (1, 1, wy1 * wx1)):
        xi, yi = x0 + dx, y0 + dy
        ok = (xi >= 0) & (xi <= W - 1) & (yi >= 0) & (yi <= H - 1) & (w != 0)
        for c in range(C):
            contrib = (go[:, c] * w).astype(np.float32).astype(np.float64)       # the fp32 product, exactly
            nn, yy, xx = np.broadcast_to(n_idx, ok.shape)[ok], yi[ok], xi[ok]
            np.add.at(ref, (nn, c, yy, xx), contrib[ok])
            np.add.at(count, (nn, c, yy, xx), 1)
    return ref, count


def _run_sampler_det(emu, go, data, grid, order):
    N, C, OH, OW = go.shape
    H, W = data.shape[2:]
    gd = np.zeros(data.shape, np.float32)
    gg = np.full((N, 2, OH, OW), np.nan, np.float32)
    emu.emu_bilinear_sampler_backward_det(_ptr(go), _ptr(data), _ptr(grid), _ptr(gd), _ptr(gg), N, C, H, W, OH, OW,
                                          _ptr(np.ascontiguousarray(order, np.int64)))
    return gd, gg


def _check_within_bound(emu, got, ref, count, bound, fanin):
    """|got - float64 sum| <= n 2^-(s+1) per element (det.cuh) plus the final rounding to fp32"""
    s, finite = _scale_exp(emu, bound, fanin)
    assert finite
    err = np.abs(got.astype(np.float64) - ref)
    allowed = count * 2.0 ** -(s + 1) + np.abs(ref) * 2.0 ** -23
    assert (err <= allowed).all(), float((err - allowed).max())
    return s


def test_fixed_point_scatter_is_order_independent_and_within_bound(emu):
    rng = np.random.default_rng(0)
    N, C, H, W, OH, OW = 2, 3, 9, 13, 11, 15
    data = rng.standard_normal((N, C, H, W)).astype(np.float32)
    xr = rng.uniform(-2, W + 1, (N, OH, OW))
    yr = rng.uniform(-2, H + 1, (N, OH, OW))
    grid = np.stack([xr / ((W - 1) / 2) - 1, yr / ((H - 1) / 2) - 1], axis=1).astype(np.float32)
    go = (rng.standard_normal((N, C, OH, OW)) * 10.0 ** rng.uniform(-3, 3, (N, C, OH, OW))).astype(np.float32)
    pix = N * OH * OW
    base_gd, base_gg = _run_sampler_det(emu, go, data, grid, np.arange(pix))
    for seed in range(4):                                    # several random thread orders, and the reverse one
        order = np.random.default_rng(100 + seed).permutation(pix) if seed < 3 else np.arange(pix)[::-1]
        gd, gg = _run_sampler_det(emu, go, data, grid, order)
        assert np.array_equal(gd.view(np.uint32), base_gd.view(np.uint32))
        assert np.array_equal(gg, base_gg)
    ref, count = _sampler_contributions(go, grid, H, W)
    assert count.max() > 4                                   # some elements gather several contributions
    _check_within_bound(emu, base_gd, ref, count, np.abs(go).max(), 4 * OH * OW)


def test_fixed_point_scatter_all_samples_on_one_pixel(emu):
    """every output pixel samples the same position: one data element per corner gathers all N*OH*OW contributions, all
    of the same sign and close to the bound -- the worst case for the fixed-point range"""
    rng = np.random.default_rng(1)
    N, C, H, W, OH, OW = 1, 2, 6, 7, 48, 64
    data = rng.standard_normal((N, C, H, W)).astype(np.float32)
    xr, yr = 3.5, 2.25                                        # corner weights 3/8, 1/8, 3/8, 1/8: exact in fp32
    grid = np.empty((N, 2, OH, OW), np.float32)
    grid[:, 0], grid[:, 1] = xr / ((W - 1) / 2) - 1, yr / ((H - 1) / 2) - 1
    go = rng.uniform(0.5, 1.0, (N, C, OH, OW)).astype(np.float32) * np.float32(3e33)
    gd, _ = _run_sampler_det(emu, go, data, grid, np.random.default_rng(2).permutation(N * OH * OW))
    ref, count = _sampler_contributions(go, grid, H, W)
    assert count.max() == OH * OW and np.isfinite(gd).all() and (gd >= 0).all()
    s = _check_within_bound(emu, gd, ref, count, np.abs(go).max(), 4 * OH * OW)
    assert ref.max() * 2.0 ** s > 2.0 ** 54                  # the int64 sums really ran close to their range (2^63)


def test_fixed_point_scatter_nan_and_inf_give_nan(emu):
    rng = np.random.default_rng(3)
    N, C, H, W, OH, OW = 1, 2, 5, 6, 5, 6
    data = rng.standard_normal((N, C, H, W)).astype(np.float32)
    grid = rng.uniform(-0.9, 0.9, (N, 2, OH, OW)).astype(np.float32)
    for bad in (np.nan, np.inf, -np.inf):
        go = rng.standard_normal((N, C, OH, OW)).astype(np.float32)
        go[0, 1, 2, 3] = bad
        gd, _ = _run_sampler_det(emu, go, data, grid, np.arange(N * OH * OW))
        assert np.isnan(gd).all(), bad
    fin = ctypes.c_int()
    emu.emu_det_scale(3e38, 3e38, 2, 10, ctypes.byref(fin))  # finite factors whose product leaves the fp32 range
    assert fin.value == 0
    emu.emu_det_scale(0.0, 0.0, 2, 10, ctypes.byref(fin))    # all-zero gradients: a finite scale
    assert fin.value == 1


def test_k4_bound_pass_on_host(emu):
    rng = np.random.default_rng(4)
    N, F, HW = 2, 5, 37
    g = rng.standard_normal((N, F, HW)).astype(np.float32)
    want = np.abs(g).sum(axis=1, dtype=np.float64).max()
    assert abs(emu.emu_pixel_abs_sum_max(_ptr(g), N, F, HW) - want) <= 1e-6 * want
    g[1, 3, 7] = np.nan
    assert np.isnan(emu.emu_pixel_abs_sum_max(_ptr(g), N, F, HW))


@pytest.mark.parametrize("layout", ["weight_partials", "plane_slices"])
def test_ordered_sum_is_order_independent(emu, layout):
    rng = np.random.default_rng(5)
    nparts, n = 37, 53
    if layout == "weight_partials":          # part[b * n + e] (K4 grad_weight), accumulated into the output
        part = rng.standard_normal((nparts, n)).astype(np.float32)
        ps, es, acc = n, 1, 1
        cols = part
    else:                                    # part[e * nparts + b] (preprocess plane sums), overwriting the output
        part = rng.standard_normal((n, nparts)).astype(np.float32)
        ps, es, acc = 1, nparts, 0
        cols = part.T
    base = rng.standard_normal(n).astype(np.float32)
    want = np.zeros(n, np.float32)
    for b in range(nparts):                  # fp32, parts in index order
        want = (want + cols[b]).astype(np.float32)
    want = (base + want).astype(np.float32) if acc else want
    for seed in range(3):
        out = base.copy()
        emu.emu_ordered_sum(_ptr(part), nparts, ps, es, _ptr(out), n, acc, _ptr(np.random.default_rng(seed).permutation(n)))
        assert np.array_equal(out, want)


def test_det_entry_points_check_the_workspace_without_gpu():
    """a null or too small det_ws returns MFN_ERR_INVALID_ARG before anything is launched; the size the library asks for
    is ops.det_workspace_bytes"""
    L = _lib.lib()
    buf = (ctypes.c_float * 64)()
    p = ctypes.cast(buf, ctypes.c_void_p)
    N, C, H, W, F = 2, 5, 12, 20, 7
    cases = {
        "mfn_warp_mask_backward_det": (lambda ws, nb: L.mfn_warp_mask_backward_det(
            *([p] * 14), N, C, H, W, F, 20.0, 8.0, 0.1, 0, ws, nb, None), ops.det_workspace_bytes("warp_mask", N, C, H, W, F)),
        "mfn_deformable_conv_backward_det": (lambda ws, nb: L.mfn_deformable_conv_backward_det(
            *([p] * 8), N, C, H, W, F, 0, ws, nb, None), ops.det_workspace_bytes("deformable_conv", N, C, H, W, F)),
        "mfn_bilinear_sampler_backward_det": (lambda ws, nb: L.mfn_bilinear_sampler_backward_det(
            *([p] * 5), N, C, H, W, 9, 11, ws, nb, None), ops.det_workspace_bytes("bilinear_sampler", N, C, H, W)),
        "mfn_image_warp_concat_backward_det": (lambda ws, nb: L.mfn_image_warp_concat_backward_det(
            *([p] * 7), N, C, H, W, 20.0, ws, nb, None), ops.det_workspace_bytes("image_warp_concat", N, C, H, W)),
        "mfn_preprocess_forward_det": (lambda ws, nb: L.mfn_preprocess_forward_det(
            p, p, 1, p, p, p, N, C, H, W, 64, 64, ws, nb, None), ops.det_workspace_bytes("preprocess", N, C, H, W)),
    }
    for name, (call, need) in cases.items():
        n0 = _lib.launch_count()
        assert call(None, 1 << 40) == -1, name
        msg = L.mfn_last_error().decode()
        assert name in msg and "null pointer" in msg and "det_ws" in msg, msg
        assert call(p, need - 1) == -1, name
        msg = L.mfn_last_error().decode()
        assert int(re.search(r"needs (\d+)", msg).group(1)) == need, (name, msg, need)
        assert _lib.launch_count() == n0
    # the counterparts' validation is unchanged
    assert L.mfn_bilinear_sampler_backward(p, None, p, p, p, 1, 1, 2, 2, 2, 2, None) == -1
    assert L.mfn_last_error() == b"mfn_bilinear_sampler_backward: null pointer"


def test_pipeline_refuses_cudnn_benchmark(monkeypatch):
    from maskflownet_b200 import pipeline
    monkeypatch.setattr(torch.backends.cudnn, "benchmark", True)
    with pytest.raises(_lib.MaskflowError, match="benchmark"):
        pipeline.PipelineFlownet(device="cpu", deterministic=True)


# ---------------------------------------------------------------------------------------------------------------
# GPU: the entry points through ops
# ---------------------------------------------------------------------------------------------------------------
DEV = "cuda"


def _cu(a, grad=False):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV).requires_grad_(grad)


def _close(got, want, tol):
    err = (got.double() - want.double()).abs().max().item()
    assert err <= tol * max(want.abs().max().item(), 1.0), (err, want.abs().max().item())


def _feat(rng, shape):
    a = rng.standard_normal(shape).astype(np.float32)
    return np.where(a > 0, a, 0.1 * a).astype(np.float32)


def _warp_mask_case(seed, N, C, F, H, W):
    """the inputs of tests/test_ops_gpu.py's warp_mask tests (level statistics, up = 2, stride 8)"""
    rng = np.random.default_rng(seed)
    x = _feat(rng, (N, C, H, W))
    w = (rng.standard_normal((F, C, 3, 3)) * np.sqrt(2.0 / (9 * C))).astype(np.float32)
    b = (rng.standard_normal(F) * 0.1).astype(np.float32)
    flow = (rng.standard_normal((N, 2, H // 2, W // 2)) * 0.4).astype(np.float32)
    mask = (rng.standard_normal((N, 1, H // 2, W // 2)) + 0.5).astype(np.float32)
    trade = (rng.standard_normal((N, F, H, W)) * 0.3).astype(np.float32)
    go = rng.standard_normal((N, F, H, W)).astype(np.float32)
    gflow = rng.standard_normal((N, 2, H, W)).astype(np.float32)
    return [x, flow, mask, w, b, trade], go, gflow


def _warp_mask_grads(arrs, go, gflow, border):
    t = [_cu(a, True) for a in arrs]
    out, fup, _ = ops.warp_mask(*t, 20.0, 8.0, 2, 0.1, border)
    ((out * _cu(go)).sum() + (fup * _cu(gflow)).sum()).backward()
    return [v.grad for v in t]


@pytest.mark.gpu
@pytest.mark.parametrize("N,C,F,H,W", [(2, 12, 12, 8, 12), (8, 32, 32, 96, 128)])   # + BASELINE configs[2] level 2
@pytest.mark.parametrize("border", [0, 1])
def test_warp_mask_backward_det(N, C, F, H, W, border):
    # the reference in fp32, like tests/test_ops_gpu.py: it rounds the sample positions as the kernels do, which matters at
    # the discontinuous MXNET15 border (a position just below 0 reads nothing, just above it reads pixel 0)
    arrs, go, gflow = _warp_mask_case(9, N, C, F, H, W)
    r = [_cu(a).requires_grad_() for a in arrs]
    with torch.device(DEV):
        ro, rf, _ = torch_ref.warp_mask(*r, 20.0, 8, 2, border)
    ((ro * _cu(go)).sum() + (rf * _cu(gflow)).sum()).backward()
    with det_mode():
        det1 = _warp_mask_grads(arrs, go, gflow, border)
        det2 = _warp_mask_grads(arrs, go, gflow, border)
    atomic = _warp_mask_grads(arrs, go, gflow, border)
    for name, a, b, c, want in zip("x flow mask w b trade".split(), det1, det2, atomic, r):
        assert torch.equal(a, b), name
        _close(a, want.grad, 2e-4)
        _close(a, c, 2e-4)


@pytest.mark.gpu
@pytest.mark.parametrize("border", [0, 1])
def test_deformable_conv_backward_det(border):
    rng = np.random.default_rng(8)
    N, C, F, H, W = 2, 10, 7, 9, 11
    arrs = [_feat(rng, (N, C, H, W)), (rng.standard_normal((N, 18, H, W)) * 1.5).astype(np.float32),
            (rng.standard_normal((F, C, 3, 3)) * 0.2).astype(np.float32), rng.standard_normal(F).astype(np.float32)]
    go = rng.standard_normal((N, F, H, W)).astype(np.float32)
    rt = [torch.from_numpy(a).clone().requires_grad_() for a in arrs]
    torch_ref.deformable_conv(*rt, border).backward(torch.from_numpy(go))

    def grads():
        t = [_cu(a, True) for a in arrs]
        ops.deformable_convolution(*t, border_mode=border).backward(_cu(go))
        return [v.grad for v in t]

    with det_mode():
        det1, det2 = grads(), grads()
    atomic = grads()
    for name, a, b, c, want in zip("x offset weight bias".split(), det1, det2, atomic, rt):
        assert torch.equal(a, b), name
        _close(a.cpu(), want.grad, 2e-4)
        _close(a, c, 2e-4)


@pytest.mark.gpu
@pytest.mark.parametrize("N,C,H,W", [(2, 3, 24, 40), (4, 3, 448, 1024)])
def test_bilinear_sampler_backward_det(N, C, H, W):
    rng = np.random.default_rng(3)
    img = rng.standard_normal((N, C, H, W)).astype(np.float32)
    pos = lambda n: rng.integers(-6, 6, (N, H, W)) + rng.uniform(0.2, 0.8, (N, H, W))
    flow_yx = np.stack([pos(H), pos(W)], axis=1).astype(np.float32)
    go = rng.standard_normal((N, C, H, W)).astype(np.float32)

    def grads():
        x, f = _cu(img, True), _cu(flow_yx, True)
        ops.reconstruction2d(x, f).backward(_cu(go))
        return [x.grad, f.grad]

    xr, fr = _cu(img).double().requires_grad_(), _cu(flow_yx).double().requires_grad_()
    with torch.device(DEV):
        torch_ref.reconstruction2d(xr, fr).backward(_cu(go).double())
    with det_mode():
        det1, det2 = grads(), grads()
    atomic = grads()
    for a, b, c, want in zip(det1, det2, atomic, (xr, fr)):
        assert torch.equal(a, b)
        _close(a, want.grad, 1e-4)
        _close(a, c, 1e-4)


@pytest.mark.gpu
@pytest.mark.parametrize("N,Ci,H,W", [(2, 3, 64, 96), (4, 3, 448, 1024)])
def test_image_warp_concat_backward_det(N, Ci, H, W):
    rng = np.random.default_rng(4)
    im1 = rng.random((N, Ci, H, W)).astype(np.float32) - 0.5
    im2 = rng.random((N, Ci, H, W)).astype(np.float32) - 0.5
    k = rng.integers(-2, 3, (N, 2, H // 4, W // 4))
    fq = ((16.0 * k + rng.uniform(0.2, 0.8, k.shape)) / 20.0).astype(np.float32)
    mq = rng.standard_normal((N, 1, H // 4, W // 4)).astype(np.float32)
    g40 = rng.standard_normal((N, Ci + 1, H, W)).astype(np.float32)

    def grads():
        a = [_cu(v, True) for v in (im2, fq, mq)]
        ops.image_warp_concat(None, *a, 20.0, want_c30=False)[1].backward(_cu(g40))
        return [v.grad for v in a]

    r = [_cu(v).double().requires_grad_() for v in (im2, fq, mq)]
    with torch.device(DEV):
        torch_ref.image_warp_concat(*r, 20.0).backward(_cu(g40).double())
    with det_mode():
        det1, det2 = grads(), grads()
    atomic = grads()
    for a, b, c, want in zip(det1, det2, atomic, r):
        assert torch.equal(a, b)
        _close(a, want.grad, 1e-4)
        _close(a, c, 1e-4)


@pytest.mark.gpu
def test_preprocess_det():
    rng = np.random.default_rng(6)
    u1 = _cu(rng.integers(0, 256, (4, 3, 436, 1024), dtype=np.uint8))
    u2 = _cu(rng.integers(0, 256, (4, 3, 436, 1024), dtype=np.uint8))
    with det_mode():
        d1, d2 = ops.preprocess(u1, u2, (448, 1024)), ops.preprocess(u1, u2, (448, 1024))
    a = ops.preprocess(u1, u2, (448, 1024))
    mean = torch.cat([u1, u2], dim=2).double().mean(dim=(2, 3), keepdim=True) / 255.0
    for x, y, z in zip(d1, d2, a):
        assert torch.equal(x, y)
        _close(x, z, 1e-5)
    _close(d1[2], mean, 1e-6)


def _record_calls(monkeypatch):
    names = []
    real = ops._call

    def rec(name, dev, *args):
        names.append(name)
        return real(name, dev, *args)

    monkeypatch.setattr(ops, "_call", rec)
    return names


def _exercise_ops():
    """forward + backward of every op that has a *_det entry point"""
    arrs, go, gflow = _warp_mask_case(1, 2, 8, 8, 8, 12)
    _warp_mask_grads(arrs, go, gflow, 0)
    x, off = torch.randn(1, 4, 6, 7, device=DEV, requires_grad=True), torch.randn(1, 18, 6, 7, device=DEV, requires_grad=True)
    w = torch.randn(5, 4, 3, 3, device=DEV, requires_grad=True)
    ops.deformable_convolution(x, off, w, no_bias=True).sum().backward()
    d, f = torch.randn(1, 3, 8, 12, device=DEV, requires_grad=True), torch.randn(1, 2, 8, 12, device=DEV, requires_grad=True)
    ops.reconstruction2d(d, f).sum().backward()
    i2, fq = torch.randn(1, 3, 16, 24, device=DEV, requires_grad=True), torch.randn(1, 2, 4, 6, device=DEV, requires_grad=True)
    mq = torch.randn(1, 1, 4, 6, device=DEV, requires_grad=True)
    ops.image_warp_concat(None, i2, fq, mq, 20.0, want_c30=False)[1].sum().backward()
    u = torch.randint(0, 256, (1, 3, 30, 40), device=DEV, dtype=torch.uint8)
    ops.preprocess(u, u, (64, 64))


DET_NAMES = {"mfn_warp_mask_backward_det", "mfn_deformable_conv_backward_det", "mfn_bilinear_sampler_backward_det",
             "mfn_image_warp_concat_backward_det", "mfn_preprocess_forward_det"}


@pytest.mark.gpu
def test_op_layer_selects_entry_points_by_the_torch_flag(monkeypatch):
    names = _record_calls(monkeypatch)
    with det_mode(False):
        _exercise_ops()
    old = list(names)
    assert not any(n.endswith("_det") for n in old)
    assert {n + "_det" for n in old} & DET_NAMES == DET_NAMES          # every counterpart was called
    for warn_only in (False, True):                                      # warn_only selects the deterministic kernels too
        names.clear()
        with det_mode(True, warn_only=warn_only):
            _exercise_ops()
        assert [n[:-4] if n in DET_NAMES else n for n in names] == old, names


# ---------------------------------------------------------------------------------------------------------------
# GPU: reproducible training in fresh processes
# ---------------------------------------------------------------------------------------------------------------
_TRAIN_SCRIPT = r"""
import json, sys
import numpy as np, torch
from maskflownet_b200 import augment, pipeline
out = sys.argv[1]
n, orig, target = 2, (288, 416), (256, 384)
rng = np.random.default_rng(7)
img1 = rng.integers(0, 256, (n, 3) + orig, dtype=np.uint8)
img2 = rng.integers(0, 256, (n, 3) + orig, dtype=np.uint8)
label = (rng.standard_normal((n, 2) + orig) * 2).astype(np.float32)
res, state = {}, {}
for cls, fix in (("MaskFlownet_S", False), ("MaskFlownet", False), ("MaskFlownet", True)):
    tag = cls + ("_fixed_head" if fix else "")
    torch.manual_seed(0)
    pipe = pipeline.PipelineFlownet(network_class=cls, deterministic=True)
    if fix:
        pipe.fix_head()
    geo = augment.GeometryAugmentation(angle_range=(-17, 17), zoom_range=(0.5, 1 / 0.9), aspect_range=(0.9, 1 / 0.9),
                                       translation_range=0.1, target_shape=target, orig_shape=orig, batch_size=n,
                                       relative_angle=0.25, relative_scale=(0.96, 1 / 0.96), relative_translation=0.25, seed=3)
    col = augment.ColorAugmentation(contrast_range=(-0.4, 0.8), brightness_sigma=0.1, channel_range=(0.8, 1.4), batch_size=n,
                                    shape=target, noise_range=(0, 0.04), saturation=0.5, hue=0.5, seed=4)
    res[tag] = [pipe.train_batch(img1, img2, label, geo, col)["epe"] for _ in range(3)]
    assert not torch.are_deterministic_algorithms_enabled()        # the pipeline restored the flag
    state.update({tag + "." + k: v.detach().cpu() for k, v in pipe.network.state_dict().items()})
    if not fix:
        v_img = [np.ascontiguousarray(a.transpose(1, 2, 0)) for a in img1]
        v_img2 = [np.ascontiguousarray(a.transpose(1, 2, 0)) for a in img2]
        v_lab = [np.ascontiguousarray(a.transpose(1, 2, 0)) for a in label]
        res[tag + "_validate"] = [pipe.validate(v_img, v_img2, v_lab, batch_size=2) for _ in range(2)]
torch.save(state, out + ".pt")
json.dump(res, open(out + ".json", "w"))
"""


@pytest.mark.gpu
def test_training_is_bit_reproducible_across_processes(tmp_path):
    """three train_batch steps of MaskFlownet-S, of the cascade with a trainable head and with a frozen one, in two fresh
    processes with the same seeds: identical losses, identical parameters (torch.equal on every tensor), and validate
    returns the identical float twice"""
    env = dict(os.environ, CUBLAS_WORKSPACE_CONFIG=":4096:8", PYTHONPATH=ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""))
    flags = ["-s"] if sys.flags.no_user_site else []
    runs = []
    for i in range(2):
        out = str(tmp_path / f"run{i}")
        r = subprocess.run([sys.executable, *flags, "-c", _TRAIN_SCRIPT, out], env=env, cwd=ROOT, capture_output=True, text=True)
        assert r.returncode == 0, r.stderr[-4000:]
        runs.append((json.load(open(out + ".json")), torch.load(out + ".pt")))
    (res0, st0), (res1, st1) = runs
    assert res0 == res1, (res0, res1)
    for tag, v in res0.items():
        assert all(np.isfinite(v)), (tag, v)
        if tag.endswith("_validate"):
            assert v[0] == v[1], (tag, v)
    assert st0.keys() == st1.keys() and len(st0) > 0
    assert all(torch.equal(st0[k], st1[k]) for k in st0), [k for k in st0 if not torch.equal(st0[k], st1[k])][:5]
