"""Every backward launch of the benchmarked training steps against float64, at the benchmark's own shapes.

bench.py --config fwdbwd (MaskFlownet-S, batch 8, 384x512) and --config train8 (batch 4 per GPU, 576x960) time the backward
kernels of the correlation (corr_bwd.cu), the fused warp (warp_bwd.cu), the transposed Upsample and the fused
MultiscaleEpe (loss.cu); the cascade adds md=2 correlations, maskless warps (one at up = 1, F = 196) and the image warp
(image_warp_bwd.cu).  Their shape decides which code runs: ragged last 32-wide tiles and the scalar store path of the
correlation at widths 15 .. 240, the 128-pixel CTA partials of g_W, the clamped last coarse row of a 9x15 Upsample(64).
So this file runs one training step per benchmarked config and checks every launch while it happens: the forward through
launchcheck.recorders.Recorder, the backward through wrappers of the autograd Functions' backward methods
(BackwardCFunction looks `backward` up on the Function class at call time).  Each wrapper runs the original, synchronises,
and compares that launch alone with a float64 reference on the GPU computed from ctx.saved_tensors and the incoming
gradient -- the values the kernel read.  The LeakyReLU masks come from the saved fp32 outputs, as the kernels take them.

Bound.  All these kernels are exact fp32 arithmetic, so per output element
    |got - ref| <= gamma_L S      gamma_L = L u / (1 - L u),  u = 2^-24
where S is the same sum with every term replaced by its absolute value and L the longest chain of fp32 roundings in the
kernel's own order, derived from the source next to each check.  This is a worst-case bound: correct fp32 arithmetic in
that order cannot exceed it, and it is small enough to see an error in a small element (a bound of max-relative form
cannot).  Additions to it, each derived where it is used:
  * the sigmoid of the mask is __expf-based (max error 2 + floor(1.173 |v|) ulp, CUDA C Programming Guide); its error
    enters as kappa S with kappa = max (1 - sig) delta_exp + 2u (relative), and in g_mask as |1 - 2 sig| times its
    absolute error;
  * deterministic mode (det.cuh): an element that receives n fixed-point contributions is off by n 2^(k+e-62) + u |ref|;
  * the image warp and the EPE read fp32 positions / up-sampled values the reference cannot reproduce bit for bit: their
    rounding (2^-20 (|p| + |d| + 1) px, gamma_5 of the interpolated values) times the slope.
The robust EPE of the KITTI / Sintel fine-tuning, e = (|d0| + |d1| + eps)^q with q = 0.4, eps = 1e-8, has a steep
gradient q s^(q-1) sign(d_c) near d = 0 (s = |d0| + |d1| + eps), so its bound is taken over the box the kernel's fp32 d can
lie in: each d_c off by delta_c = gamma_6 (max |pred| + |flow_c|), s in [s_lo, s_hi], widened by powf's error.  Where
|d_c| <= delta_c the sign is open; where s_lo reaches eps the bound is rigorous but says little, and the fraction of such
gradient elements is reported and asserted small (epe_backward_bounds, test_dataset_shapes_backward.py).
The image warp's backward is checked on what the cascade's graph asks of it: g_mask_up, g_im2 where the image requires a
gradient, and g_flow_up where the flow does (the cascade trained end to end).  The flow gradient is the sampler's slope,
which jumps where the position crosses an integer: an fp32 position within its rounding bound of an integer may take
either cell's slope, and is accepted against either (image_warp_flow_slopes).
The cuDNN convolution backward (ops._Conv3x3TrainFn) is not this library's arithmetic: only its wiring is checked (mask from
the saved y, stride, dilation, padding, bias) against float64 autograd at 2^-12 (S + 2^-8 max S): cuDNN's transform
algorithms leave rounding noise where the exact gradient is 0, which a wiring error (O(S) everywhere) is far above.

Sensitivity is asserted (each control must fail the bound by CONTROL_MARGIN on one real launch of each kind) and so is
coverage (launch counts per kind equal the graph's; the deterministic run calls the *_det entry points only).
test_bound_accepts_emulated_kernel_order_and_rejects_controls checks the bound on the CPU against the kernels' summation
orders emulated in fp32.  One line per launch is printed (pytest -s): err / bound and err / (u S).
"""
import math
import time

import pytest
import torch
import torch.nn.functional as tF

from maskflownet_b200 import losses, network, ops
from oracle import torch_ref

from launchcheck import fp64_references  # noqa: F401
from launchcheck.backward import (TAPS, _f32, _gather0, _tap_positions, corr_bwd_ref, epe_backward_bounds, epe_delta,
                                  epe_forward_bound, epe_q_controls, image_warp_flow_slopes, judge_bound, warp_bwd_S,
                                  warp_bwd_ref)
from launchcheck.bounds import CONTROL_MARGIN
from launchcheck.inputs import _images_u8, _named_model
from launchcheck.recorders import BackwardRecorder, Recorder


# ------------------------------------------------------------------------------------------------------------------
# CPU: the bound accepts the kernels' summation orders and rejects the controls
# ------------------------------------------------------------------------------------------------------------------
def test_bound_accepts_emulated_kernel_order_and_rejects_controls():
    g = torch.Generator().manual_seed(11)
    # ---- correlation backward, side A: acc = fma chain over the (ey, ex) stencil, then * fl(1 / C) -------------------
    md, C, H, W = 4, 32, 7, 37
    D = (2 * md + 1) ** 2
    f1, f2 = torch.randn((1, C, H, W), generator=g), torch.randn((1, C, H, W), generator=g)
    go, res = torch.randn((1, D, H, W), generator=g), torch.randn((1, D, H, W), generator=g)
    slope = _f32(0.1)
    gp = torch.where(res > 0, go, go * torch.tensor(0.1, dtype=torch.float32))          # fp32, as the kernel loads it
    pad = tF.pad(f2, (md, md, md, md))
    acc = torch.zeros((1, C, H, W))
    for q in range(D):
        ey, ex = q // (2 * md + 1), q % (2 * md + 1)
        acc = (acc + gp[:, q:q + 1] * pad[:, :, ey:ey + H, ex:ex + W]).float()
    got = acc * torch.tensor(1.0 / C, dtype=torch.float32)
    g1, _, s1, _ = corr_bwd_ref(f1, f2, gp.double(), md)
    r, _, _ = judge_bound(got, g1, s1, D + 3)
    assert r <= 1.0, r
    gp_drop = gp.double().clone()
    gp_drop[:, 0] = 0
    no_leaky = go.double()
    for name, alt in (("plane", gp_drop), ("leaky", no_leaky)):
        c1 = corr_bwd_ref(f1, f2, alt, md)[0]
        assert judge_bound(c1, g1, s1, D + 3)[0] >= CONTROL_MARGIN, name

    # ---- K4 g_W and g_b: 128-pixel partials (fma chain per CTA), then the CTA partials added in sequence ----------------
    N, C, F, H, W = 2, 4, 3, 20, 29
    P = N * H * W
    gconv = torch.randn((P, F), generator=g)
    samp = torch.randn((P, C * 9), generator=g)
    parts = []
    for p0 in range(0, P, 128):
        a = torch.zeros((F, C * 9))
        for q in range(p0, min(p0 + 128, P)):
            a = (a + gconv[q].view(F, 1) * samp[q].view(1, -1)).float()
        parts.append(a)
    gw = torch.zeros((F, C * 9))
    for a in parts:
        gw = (gw + a).float()
    ref = gconv.double().t() @ samp.double()
    S = gconv.double().abs().t() @ samp.double().abs()
    L_w = 128 + math.ceil(P / 128) + 10
    assert judge_bound(gw, ref, S, L_w)[0] <= 1.0
    last = gconv.double()[-(P - 128 * (len(parts) - 1)):].t() @ samp.double()[-(P - 128 * (len(parts) - 1)):]
    assert judge_bound(ref - last, ref, S, L_w)[0] >= CONTROL_MARGIN
    lanes = torch.zeros((256, F))                 # plane_sum: thread t adds pixels t, t + 256, ... in turn
    for p0 in range(0, P, 256):
        blk = gconv[p0:p0 + 256]
        lanes[:blk.shape[0]] = (lanes[:blk.shape[0]] + blk).float()
    while lanes.shape[0] > 1:                        # the shuffle trees
        lanes = (lanes[0::2] + lanes[1::2]).float()
    gb = lanes[0]
    L_b = N * math.ceil(H * W / 256) + 16
    gb_ref, gb_S = gconv.double().sum(0), gconv.double().abs().sum(0)
    assert judge_bound(gb, gb_ref, gb_S, L_b)[0] <= 1.0
    assert judge_bound(gb_ref - gconv.double()[128 * (len(parts) - 1):].sum(0), gb_ref, gb_S, L_b)[0] >= CONTROL_MARGIN

    # ---- K4 flow gradient: gS = sum_f W g (chain over f), th = sum_c gS * slope, gdy = sum over taps ------------------
    N, C, F, H, W = 1, 8, 6, 9, 13
    x = torch.randn((N, C, H, W), generator=g)
    w = torch.randn((F, C, 3, 3), generator=g) * 0.3
    gc = torch.randn((N, F, H, W), generator=g)
    fup = torch.randn((N, 2, H, W), generator=g) * 1.5
    fup[:, 0, -2:] = 0.9 * 32 / 20          # rows whose lower taps land in the collapsed band [H - 1, H)
    scale, stride, border = 20.0, 32.0, ops.BORDER_MXNET15
    k32 = torch.tensor(scale / stride, dtype=torch.float32)
    gdy = torch.zeros((N, H, W))
    for i, j in TAPS:
        h, v = _tap_positions(fup, scale, stride, i, j)
        hl = h.clone().requires_grad_()
        th = torch.zeros((N, H, W))
        for c in range(C):
            gS = torch.zeros((N, H, W))
            for f in range(F):
                gS = (gS + w[f, c, i, j] * gc[:, f]).float()
            sl = torch.autograd.grad(torch_ref.sample_tap(x[:, c:c + 1].double(), hl, v, border).sum(), hl)[0]
            th = (th + gS * sl.float()).float()
        gdy = (gdy + th).float()
    got = (gdy * k32).float()
    gx_ref, gf_ref, _ = warp_bwd_ref(x, fup, w, gc.double(), scale, stride, border)
    _, Sf, _ = warp_bwd_S(x, fup, w, gc.double().abs(), scale, stride, border)
    L_f = F + 9 * C + 9
    assert judge_bound(got, gf_ref[:, 0], Sf[:, 0], L_f)[0] <= 1.0
    tap0 = warp_bwd_ref(x, fup, w, gc.double(), scale, stride, border, taps=((0, 0),))
    assert judge_bound(gf_ref - tap0[1], gf_ref, Sf, L_f)[0] >= CONTROL_MARGIN
    Sgx, _, _ = warp_bwd_S(x, fup, w, gc.double().abs(), scale, stride, border)
    assert judge_bound(gx_ref - tap0[0], gx_ref, Sgx, F + 8 + 36)[0] >= CONTROL_MARGIN
    # the emulated shape reaches the MXNet-1.5 collapsed band, where the reference's slope is zero
    h, _ = _tap_positions(fup, scale, stride, 2, 1)
    assert bool((torch.floor(h) >= H - 1).any())


def _emu_upsample(p, s, H, W):
    """Upsample(s) of p (N, C, H / s, W / s) in the kernels' fp32 order (upsample_at, sampling.cuh), one rounding per
    operation."""
    Hc, Wc = p.shape[2:]
    y, x = torch.arange(H), torch.arange(W)
    y0, x0 = y // s, x // s
    y1, x1 = (y0 + 1).clamp(max=Hc - 1), (x0 + 1).clamp(max=Wc - 1)
    wy = ((y - y0 * s).float() / s).view(H, 1)
    wx = ((x - x0 * s).float() / s).view(1, W)
    a, b = p[:, :, y0][:, :, :, x0], p[:, :, y0][:, :, :, x1]
    c, d = p[:, :, y1][:, :, :, x0], p[:, :, y1][:, :, :, x1]
    top, bot = a + (b - a) * wx, c + (d - c) * wx
    return top + (bot - top) * wy


def _emu_lanes(v):
    """The sum of v (fp32, 1-D) as 32 lanes add it (lane l takes elements l, l + 32, ...) and a xor shuffle tree."""
    lanes = torch.zeros(32)
    for k in range(0, v.numel(), 32):
        blk = v[k:k + 32]
        lanes[:blk.numel()] = lanes[:blk.numel()] + blk
    idx = torch.arange(32)
    for o in (16, 8, 4, 2, 1):
        lanes = lanes + lanes[idx ^ o]
    return lanes[0]


def _emu_epe(flow, mask, preds, scales, weights, eps, q, gl):
    """epe_forward_kernel + epe_finish_kernel and epe_backward_kernel (loss.cu) for one sample, H W <= 16384, in fp32."""
    N, _, H, W = flow.shape
    assert N == 1 and H * W <= 16384
    eps32, q32 = torch.tensor(eps, dtype=torch.float32), torch.tensor(q, dtype=torch.float32)
    ups = [_emu_upsample(p, s, H, W) for p, s in zip(preds, scales)]
    e = torch.zeros((H, W))
    kg = []
    for u, w in zip(ups, weights):
        d = u[0] - flow[0]
        sv = d[0].abs() + d[1].abs() + eps32
        e = e + torch.tensor(w, dtype=torch.float32) * sv ** q32
        k = q32 * sv ** (q32 - 1)
        kg.append(torch.stack([torch.where(d[c] > 0, k, torch.where(d[c] < 0, -k, torch.zeros_like(k))) for c in (0, 1)]))
    # forward: thread t of block b holds pixel 256 b + t; warp trees, the block's warps in order, the blocks in order
    parts = torch.zeros((2, 64 * 256))
    parts[0, :H * W], parts[1, :H * W] = (e * mask[0, 0]).reshape(-1), mask[0, 0].reshape(-1)
    parts = parts.view(2, 64, 8, 32)
    idx = torch.arange(32)
    for o in (16, 8, 4, 2, 1):
        parts = parts + parts[..., idx ^ o]
    num, den = torch.zeros(()), torch.zeros(())
    for b in range(64):
        bn, bd = torch.zeros(()), torch.zeros(())
        for wp in range(8):
            bn, bd = bn + parts[0, b, wp, 0], bd + parts[1, b, wp, 0]
        num, den = num + bn, den + bd
    loss = (num / den).view(1)
    # backward: one warp per coarse pixel over the full-resolution pixels that read it
    grads = []
    for p, s, w, g in zip(preds, scales, weights, kg):
        Hc, Wc = p.shape[2:]
        out = torch.zeros_like(p)
        kk = torch.tensor(w, dtype=torch.float32) * gl[0] / den
        for i in range(Hc):
            for j in range(Wc):
                ys = torch.arange(max(s * (i - 1), 0), min(s * (i + 1), H))
                xs = torch.arange(max(s * (j - 1), 0), min(s * (j + 1), W))
                y0, x0 = ys // s, xs // s
                y1, x1 = (y0 + 1).clamp(max=Hc - 1), (x0 + 1).clamp(max=Wc - 1)
                wy, wx = (ys - y0 * s).float() / s, (xs - x0 * s).float() / s
                cy = torch.where(y0 == i, 1 - wy, torch.zeros_like(wy)) + torch.where(y1 == i, wy, torch.zeros_like(wy))
                cx = torch.where(x0 == j, 1 - wx, torch.zeros_like(wx)) + torch.where(x1 == j, wx, torch.zeros_like(wx))
                coef = (cy.view(-1, 1) * cx.view(1, -1)) * mask[0, 0][ys][:, xs]
                for c in (0, 1):
                    out[0, c, i, j] = _emu_lanes((coef * g[c][ys][:, xs]).reshape(-1)) * kk
        grads.append(out)
    return loss, den.view(1), grads


def _emu_image_warp_flow(img, fy, fx, g, scale):
    """grad_flow_up of image_warp_concat_bwd_kernel (sampler_corners, sample_backward) in fp32, given the kernel's fp32
    displacements fy, fx (N, H, W)."""
    N, C, H, W = img.shape
    yr = torch.arange(H, dtype=torch.float32).view(1, H, 1) + fy
    xr = torch.arange(W, dtype=torch.float32).view(1, 1, W) + fx
    y0, x0 = torch.floor(yr), torch.floor(xr)
    wx0, wy0 = 1 - (xr - x0), 1 - (yr - y0)
    wx1, wy1 = 1 - wx0, 1 - wy0
    y0, x0 = y0.long(), x0.long()
    xin = [(x0 + k >= 0) & (x0 + k <= W - 1) for k in (0, 1)]
    yin = [(y0 + k >= 0) & (y0 + k <= H - 1) for k in (0, 1)]
    z = torch.zeros_like(wx0)
    corners = [(0, 0), (0, 1), (1, 0), (1, 1)]
    dwx = [torch.where(xin[b] & yin[a], (wy0 if a == 0 else wy1) * (1 if b else -1), z) for a, b in corners]
    dwy = [torch.where(xin[b] & yin[a], (wx0 if b == 0 else wx1) * (1 if a else -1), z) for a, b in corners]
    vals = [_gather0(img, y0 + a, x0 + b) for a, b in corners]
    ax, ay = torch.zeros_like(z), torch.zeros_like(z)
    for c in range(C):
        sx, sy = torch.zeros_like(z), torch.zeros_like(z)
        for t in range(4):
            sx = sx + dwx[t] * vals[t][:, c]
            sy = sy + dwy[t] * vals[t][:, c]
        ax, ay = ax + g[:, c] * sx, ay + g[:, c] * sy
    return torch.stack([ay * scale, ax * scale], 1)


def test_bound_accepts_emulated_q_loss_and_flow_slope_and_rejects_controls():
    """The robust loss (q = 0.4, eps = 1e-8) and the image warp's flow gradient: the bounds accept the kernels' fp32
    arithmetic at the edges (d within delta of 0, d exactly 0 so that s = eps, positions one ulp either side of an
    integer) and reject each near miss by CONTROL_MARGIN."""
    g = torch.Generator().manual_seed(12)
    # ---- MultiscaleEpe, q form -------------------------------------------------------------------------------------
    H, W, scales, weights, q, eps = 32, 48, (8, 4), (0.08, 0.32), 0.4, _f32(1e-8)
    preds = [torch.randn((1, 2, H // s, W // s), generator=g) * 2 for s in scales]
    flow = torch.randn((1, 2, H, W), generator=g) * 2
    flow[..., W // 2:] *= 3                 # larger errors where the mask is below 1/2: rounding it moves the mean
    mask = torch.rand((1, 1, H, W), generator=g) * 0.5
    mask[..., :W // 2] += 0.5
    mask[mask < 0.1] = 0
    mask[:, :, :6, :] = 1.0
    u4 = _emu_upsample(preds[1], 4, H, W)
    zero = torch.zeros((1, 1, H, W), dtype=torch.bool)
    zero[:, :, 16:28, 8:28] = True                               # d exactly 0 at scale 4: s = eps
    flow = torch.where(zero, u4, flow)
    flow[:, :, :6, ::3] = torch.nextafter(u4[:, :, :6, ::3], torch.tensor(float("inf")))   # d one ulp from 0
    flow[:, :, :6, 1::3] = torch.nextafter(u4[:, :, :6, 1::3], torch.tensor(-float("inf")))
    gl = torch.tensor([1.0])
    loss, msum, grads = _emu_epe(flow, mask, preds, scales, weights, eps, q, gl)
    zero_s = (4, zero)
    fb = epe_forward_bound(flow, mask, preds, scales, weights, eps, q, zero_s)
    assert judge_bound(loss, *fb)[0] <= 1.0
    bb = epe_backward_bounds(flow, mask, msum, preds, scales, weights, eps, q, gl, zero_s)
    for got, (ref, S, pos, L, _) in zip(grads, bb):
        assert judge_bound(got, ref, S, L, pos)[0] <= 1.0
    # the near-zero band really is within delta of 0 there (its sign is open), the patch really has s = eps
    d4 = torch_ref.upsample(preds[1].double(), 4) - flow.double()
    near = (d4.abs() <= epe_delta(preds[1], flow, 4))[:, :, :6]
    assert bool(near[..., 0::3].all() and near[..., 1::3].all())
    assert bool((_emu_upsample(preds[1], 4, H, W) - flow)[zero.expand(-1, 2, -1, -1)].eq(0).all())
    fc = epe_q_controls(flow, mask, None, preds, scales, weights, eps, q, None, zero_s, fb, loss=loss)
    bc = epe_q_controls(flow, mask, msum, preds, scales, weights, eps, q, gl, zero_s, bb)
    assert set(fc) == {"L2 form", "mask rounded"} and set(bc) == {"L2 form", "mask rounded", "sign(0) = +1"}
    for name, r in list(fc.items()) + list(bc.items()):
        assert r >= CONTROL_MARGIN, (name, r)

    # ---- image warp: g_flow_up at fp32 positions on, and one ulp either side of, integers ---------------------------
    N, C, H, W, scale = 1, 3, 12, 16, 20.0
    img = torch.randn((N, C, H, W), generator=g)
    gout = torch.randn((N, C, H, W), generator=g)
    fy = torch.randn((N, H, W), generator=g) * 3
    fx = torch.randn((N, H, W), generator=g) * 3
    ys = torch.arange(H, dtype=torch.float32).view(1, H, 1)
    xs = torch.arange(W, dtype=torch.float32).view(1, 1, W)
    ty, tx = torch.round(ys + fy), torch.round(xs + fx)         # the nearest integer positions
    fy[:, 0::3] = (ty - ys)[:, 0::3]                                # on an integer
    fy[:, 1::3] = torch.nextafter(ty - ys, torch.tensor(float("inf")))[:, 1::3]        # one ulp either side
    fy[:, 2::3] = torch.nextafter(ty - ys, torch.tensor(-float("inf")))[:, 2::3]
    fx[:, :, 0::2] = torch.nextafter(tx - xs, torch.tensor(-float("inf")))[:, :, 0::2]
    fy[:, 5, :] = 2 - 2.0 ** -22                    # 5 + (2 - 2^-22) rounds to 7 in fp32: the float64 cell is 6
    got = _emu_image_warp_flow(img, fy, fx, gout, scale)
    h, v = ys.double() + fy.double(), xs.double() + fx.double()
    dh, dv = 2.0 ** -20 * (ys.double() + fy.double().abs() + 1), 2.0 ** -20 * (xs.double() + fx.double().abs() + 1)
    assert bool((torch.floor(h) != torch.floor(ys + fy).double()).any())     # the fp32 position took the other cell
    r, ctl, _ = image_warp_flow_slopes(img, h, v, dh, dv, gout, scale, got)
    assert r <= 1.0, r
    assert ctl >= CONTROL_MARGIN, ctl


# ------------------------------------------------------------------------------------------------------------------
# GPU: the backward recorder
# ------------------------------------------------------------------------------------------------------------------
RUNS = {   # run: (model class, batch, H, W, image seed, label seed, masked rows from the bottom, deterministic)
    "fwdbwd": (network.MaskFlownetS, 8, 384, 512, 31, 7, 0, False),
    "train8": (network.MaskFlownetS, 4, 576, 960, 32, 8, 36, False),
    "fwdbwd-det": (network.MaskFlownetS, 8, 384, 512, 31, 7, 0, True),
    "cascade-train": (network.MaskFlownet, 2, 384, 512, 33, 9, 0, False),
}


@pytest.mark.gpu
@pytest.mark.parametrize("run", list(RUNS))
@pytest.mark.usefixtures("fp64_references")
def test_every_backward_launch_of_the_benchmarked_step_against_float64(run, monkeypatch):
    cls, N, H, W, seed, lseed, band, det = RUNS[run]
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    fwd = Recorder(monkeypatch, run)
    bwd = BackwardRecorder(monkeypatch, run)
    model = _named_model(cls).train()
    u1, u2 = _images_u8(seed=seed, n=N, h=H, w=W)
    g = torch.Generator().manual_seed(lseed)
    label = (torch.randn(N, 2, H, W, generator=g) * 3).cuda()
    mask = torch.ones(N, 1, H, W, device="cuda")
    if band:
        mask[:, :, H - band:] = 0          # a 540-row frame padded to 576 rows
    prev, prev_warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(det, warn_only=True)
    try:
        a, b, _ = network.centralize(u1.float() / 255.0, u2.float() / 255.0)
        preds = model(a, b)[0]
        losses.multiscale_epe(label, mask, preds).sum().backward()
        torch.cuda.synchronize()
    finally:
        torch.use_deterministic_algorithms(prev, warn_only=prev_warn)
    secs, peak = time.perf_counter() - t0, torch.cuda.max_memory_allocated() / 2 ** 30
    monkeypatch.undo()
    fwd.report()
    bwd.report()
    print(f"{run}: {len(fwd.rows)} forward and {len(bwd.rows)} backward checks in {secs:.1f} s, peak {peak:.2f} GiB")
    assert not fwd.failures, "\n".join(fwd.failures)
    assert not bwd.failures, "\n".join(bwd.failures)

    # coverage: the graph's launch counts
    corr = [r for r in bwd.rows if r["op"] == "corr_bwd"]
    warps = bwd.calls.count("mfn_warp_mask_backward") + bwd.calls.count("mfn_warp_mask_backward_det")
    ups = [r for r in bwd.rows if r["op"] == "upsample_bwd"]
    convs_fwd = [r for r in fwd.rows if r["op"] == "conv3x3_slices"]
    convs_bwd = [r for r in bwd.rows if r["op"] == "conv_bwd"]
    cascade = cls is network.MaskFlownet
    assert len(corr) == 5 + (10 if cascade else 0), len(corr)
    assert sum(r["name"] == "md=2" for r in corr) == (10 if cascade else 0)
    assert warps == 4 + (5 if cascade else 0), warps
    assert len(ups) == 8 + (7 if cascade else 0), len(ups)
    assert sum(r["op"] == "epe_bwd" for r in bwd.rows) == 5 and sum(r["op"] == "epe_fwd" for r in bwd.rows) == 1
    assert len(convs_bwd) == len(convs_fwd), (len(convs_bwd), len(convs_fwd))
    if not cascade:
        assert len(convs_fwd) == 2 * 18 + 5 * 5 + 9 + 4 + 7
    iw = bwd.calls.count("mfn_image_warp_concat_backward") + bwd.calls.count("mfn_image_warp_concat_backward_det")
    assert iw == (1 if cascade else 0), iw
    if cascade:
        assert any(r["op"] == "warp_bwd" and r["name"].startswith("F=196 up=1") for r in bwd.rows)
        assert any(r["op"] == "image_warp_bwd" for r in bwd.rows)
        assert any(r["op"] == "image_warp_bwd" and r["name"] == "g_flow_up" for r in bwd.rows)
    if det:
        assert bwd.calls.count("mfn_warp_mask_backward_det") == 4
        atomic = {"mfn_warp_mask_backward", "mfn_deformable_conv_backward", "mfn_bilinear_sampler_backward",
                  "mfn_image_warp_concat_backward"}
        assert not atomic & set(bwd.calls), sorted(atomic & set(bwd.calls))

    # sensitivity: every control fails the bound by CONTROL_MARGIN on its launch
    want = {"corr md=4", "corr leaky", "upsample x2", "warp", "epe x64", "conv wiring"} | \
        ({"corr md=2", "image warp"} if cascade else set())
    assert want <= set(bwd.controls), sorted(bwd.controls)
    for kind, lst in bwd.controls.items():
        for entry in lst:
            assert min(entry[-1].values()) >= CONTROL_MARGIN, (kind, entry)
    want_ctl = {"g_x", "g_flow", "g_W", "g_b"} | ({"g_mask"} if not cascade else set())
    assert want_ctl <= set(bwd.controls["warp"][0][-1]), bwd.controls["warp"]
