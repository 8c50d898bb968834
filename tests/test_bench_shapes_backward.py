"""Every backward launch of the benchmarked training steps against float64, at the benchmark's own shapes.

bench.py --config fwdbwd (MaskFlownet-S, batch 8, 384x512) and --config train8 (batch 4 per GPU, 576x960) time the backward
kernels of the correlation (corr_bwd.cu), the fused warp (warp_bwd.cu), the transposed Upsample and the fused
MultiscaleEpe (loss.cu); the cascade adds md=2 correlations, maskless warps (one at up = 1, F = 196) and the image warp
(image_warp_bwd.cu).  Their shape decides which code runs: ragged last 32-wide tiles and the scalar store path of the
correlation at widths 15 .. 240, the 128-pixel CTA partials of g_W, the clamped last coarse row of a 9x15 Upsample(64).
So this file runs one training step per benchmarked config and checks every launch while it happens: the forward through
the recorder of test_bench_shapes.py, the backward through wrappers of the autograd Functions' backward methods
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
from test_bench_shapes import Recorder, _fp32_positions, _images_u8, _named_model, _ratio, _warp_offsets

U = 2.0 ** -24
# powf is within 4 ulp over its full range (CUDA C Programming Guide, "Mathematical Functions": single-precision maximum
# ulp errors); one ulp of a normal result is at most 2^-23 of it
POWF_REL = 4 * 2.0 ** -23
CONTROL_MARGIN = 3.0
EPS_WIRING = 2.0 ** -12
TAPS = tuple((i, j) for i in range(3) for j in range(3))


def gamma(L):
    return L * U / (1 - L * U)


def judge_bound(got, ref, S, L, extra=0.0):
    """(max |got - ref| / (gamma_L S + extra), max |got - ref| / (u S), flat index of the worst element)."""
    err = (got.double() - ref).abs()
    r = _ratio(err, gamma(L) * S + extra)
    i = int(torch.argmax(r))
    return float(r.reshape(-1)[i]), float(_ratio(err, U * S).max()), i


def _f32(v):
    return float(torch.tensor(v, dtype=torch.float32))


# ------------------------------------------------------------------------------------------------------------------
# float64 references (any device)
# ------------------------------------------------------------------------------------------------------------------
def corr_bwd_ref(f1, f2, gp, md):
    """Gradients of sum(gp * correlation(f1, f2)) (float64), and their S (the same sums of absolute values)."""
    with torch.enable_grad():
        a, b = f1.double().requires_grad_(), f2.double().requires_grad_()
        g1, g2 = torch.autograd.grad(torch_ref.correlation(a, b, md), (a, b), gp)
        a, b = f1.double().abs().requires_grad_(), f2.double().abs().requires_grad_()
        s1, s2 = torch.autograd.grad(torch_ref.correlation(a, b, md), (a, b), gp.abs())
    return g1, g2, s1, s2


def _tap_positions(fup, scale, stride, i, j):
    """fp32 tap positions fl((y - 1 + i) + d), fl((x - 1 + j) + d) of the fused warp (float64 values, (N, H, W))."""
    N, _, H, W = fup.shape
    dy, dx = _warp_offsets(fup, scale, stride)
    ys = torch.arange(H, dtype=torch.float64, device=fup.device).view(1, H, 1)
    xs = torch.arange(W, dtype=torch.float64, device=fup.device).view(1, 1, W)
    return _fp32_positions(ys + (i - 1), dy), _fp32_positions(xs + (j - 1), dx)


@torch.enable_grad()
def warp_bwd_ref(x, fup, w, gconv, scale, stride, border, taps=TAPS):
    """float64 gradients (g_x, g_flow, g_W) of sum(gconv * deform(x)) at the kernel's fp32 tap positions.  The positions
    carry the derivative scale / stride (p = p_fp32 + (d64 - d64.detach())), so autograd through sample_tap gives both
    border rules' one-sided slopes, the collapsed MXNet-1.5 row included."""
    xg, wg, fg = x.double().requires_grad_(), w.double().requires_grad_(), fup.double().requires_grad_()
    k = scale / stride
    ddy, ddx = fg[:, 0] * k, fg[:, 1] * k
    out = 0
    for i, j in taps:
        h, v = _tap_positions(fup, scale, stride, i, j)
        h, v = h + (ddy - ddy.detach()), v + (ddx - ddx.detach())
        out = out + torch.einsum("fc,nchw->nfhw", wg[:, :, i, j], torch_ref.sample_tap(xg, h, v, border))
    return torch.autograd.grad(out, (xg, fg, wg), gconv)


@torch.enable_grad()
def warp_bwd_S(x, fup, w, gabs, scale, stride, border):
    """S of g_x, g_W (autograd of the same operator on |x|, |W|, |g_conv|) and of the coordinate gradient.  The corner
    slopes of the latter carry signs, so its S is written out per tap: |x| sampled at the two bracketing rows (columns),
    A + B = 2T + (1 - 2l) dT/dl with T = sum_c G_c sample(|x_c|), G_c = sum_f |W_fc| |g_conv_f|; zero where the MXNet-1.5
    rule collapses the axis (the kernel's slope is zero there)."""
    N, C, H, W = x.shape
    xa, wa = x.double().abs().requires_grad_(), w.double().abs().requires_grad_()
    out = 0
    sy = sx = 0
    for i, j in TAPS:
        h, v = _tap_positions(fup, scale, stride, i, j)
        out = out + torch.einsum("fc,nchw->nfhw", wa[:, :, i, j], torch_ref.sample_tap(xa, h, v, border))
        hl, vl = h.clone().requires_grad_(), v.clone().requires_grad_()
        G = torch.einsum("fc,nfhw->nchw", wa[:, :, i, j].detach(), gabs)
        T = (G * torch_ref.sample_tap(xa.detach(), hl, vl, border)).sum(1)
        dth, dtw = torch.autograd.grad(T.sum(), (hl, vl))
        T = T.detach()
        ah = 2 * T + (1 - 2 * (h - torch.floor(h))) * dth
        aw = 2 * T + (1 - 2 * (v - torch.floor(v))) * dtw
        if border == ops.BORDER_MXNET15:
            ah, aw = ah * (torch.floor(h) < H - 1), aw * (torch.floor(v) < W - 1)
        sy, sx = sy + ah, sx + aw
    sgx, sgw = torch.autograd.grad(out, (xa, wa), gabs)
    return sgx, torch.stack([sy, sx], 1) * abs(scale / stride), sgw


def corner_scatter(vals, h, v, H, W):
    """sum of vals (N, OH, OW) scattered onto the four corners of each real position (h, v), clamped into the (H, W)
    plane; positions outside (-1, H) x (-1, W) scatter nothing.  With vals = 1: an upper bound of the contributions an
    element receives."""
    N = h.shape[0]
    inside = ((h > -1) & (h < H) & (v > -1) & (v < W)).to(vals.dtype) * vals
    h0, v0 = torch.floor(h).long(), torch.floor(v).long()
    acc = torch.zeros((N, H * W), dtype=vals.dtype, device=vals.device)
    for a in (0, 1):
        for b in (0, 1):
            idx = (h0 + a).clamp(0, H - 1) * W + (v0 + b).clamp(0, W - 1)
            acc.scatter_add_(1, idx.reshape(N, -1), inside.reshape(N, -1))
    return acc.view(N, 1, H, W)


@torch.enable_grad()
def upsample_T(t, f, H, W):
    """The transposed Upsample(f) of t (N, C, fH, fW) in float64: the backward's reference (nonnegative weights, so it
    also gives S on |t|)."""
    z = torch.zeros((t.shape[0], t.shape[1], H, W), dtype=torch.float64, device=t.device, requires_grad=True)
    return torch.autograd.grad(torch_ref.upsample(z, f), z, t.double())[0]


def sigmoid_error(v):
    """(sig, absolute error bound of sigmoidf_ = 1 / (1 + __expf(-v))): __expf is within 2 + floor(1.173 |v|) ulp."""
    s = torch.sigmoid(v)
    d_exp = (2 + torch.floor(1.173 * v.abs())) * 2.0 ** -23
    return s, s * (1 - s) * d_exp + 2 * U * s


# ---- fused MultiscaleEpe (loss.cu) -----------------------------------------------------------------------------------
def epe_terms(flow, mask, preds, scales, weights, eps, q, zero=None):
    """float64 per-sample loss; per scale the up-sampled prediction u and the per-pixel EPE e.  q < 0: the L2 form
    sqrt(|d|^2 + eps); q >= 0: the robust form (|d0| + |d1| + eps)^q, whose autograd takes sign(0) = 0 as the kernel does.
    zero = (scale, bool (N, 1, H, W)): pixels where the kernel's d is exactly 0 at that scale (u is the label there)."""
    f64, m64 = flow.double(), mask.double()
    loss, parts = 0, []
    for p, s, w in zip(preds, scales, weights):
        u = torch_ref.upsample(p, s)
        if zero is not None and s == zero[0]:
            u = torch.where(zero[1], f64, u)
        if q < 0:
            e = torch.sqrt(((u - f64) ** 2).sum(1, keepdim=True) + eps)
        else:
            e = ((u - f64).abs().sum(1, keepdim=True) + eps) ** q
        loss = loss + w * (e * m64).sum(dim=(1, 2, 3))
        parts.append((u, e))
    return loss / m64.sum(dim=(1, 2, 3)), parts


def epe_delta(p, flow, s, zero=None):
    """delta_c = gamma_6 (max |pred| + |flow_c|): how far the kernel's fp32 d = Upsample(s)(pred) - flow (5 roundings of
    the interpolation, 1 of the difference) can lie from the float64 one; 0 where d is known to be exactly 0."""
    M = p.abs().amax(dim=(1, 2, 3), keepdim=True).double()
    delta = gamma(6) * (M + flow.double().abs())
    if zero is not None and s == zero[0]:
        delta = delta * ~zero[1]
    return delta


def epe_q_box(d, delta, eps):
    """The robust EPE's s = |d0| + |d1| + eps (float64, (N, 1, H, W)) and the box [s_lo, s_hi] of the kernel's
    fl(fl(|d0'| + |d1'|) + eps) when |d_c' - d_c| <= delta_c: the two additions round (gamma_2), and a rounded sum of
    nonnegative terms and eps cannot fall below eps."""
    s = d.abs().sum(1, keepdim=True) + eps
    dd = delta.sum(1, keepdim=True)
    return s, torch.clamp((s - dd) * (1 - gamma(2)), min=eps), (s + dd) * (1 + gamma(2))


def epe_forward_bound(flow, mask, preds, scales, weights, eps, q, zero=None):
    """(ref, S, L, extra) of epe_forward_kernel + epe_finish_kernel: |loss - ref| <= gamma_L S + extra.
    Per pixel: Upsample(s) (5 roundings each), d, d^2, sum, + eps, sqrt (5), * w_s, sum over scales (2 per scale); then a
    thread's ceil(HW / (64 * 256)) pixels, * mask, two reductions of 5 + 8 (block) and 64 (finish), the division:
    L = 15 * scales + ceil(HW / 16384) + 80.  The up-sampled prediction's rounding: for the L2 form (|de/du| <= 1)
    gamma_5 max |pred| twice; for the q form e is in [s_lo^q, s_hi^q] widened by powf's error, per pixel."""
    N, _, H, W = flow.shape
    ref, parts = epe_terms(flow, mask, [p.double() for p in preds], scales, weights, eps, q, zero)
    m64, f64 = mask.double(), flow.double()
    msum = m64.sum(dim=(1, 2, 3))
    L = 15 * len(preds) + math.ceil(H * W / 16384) + 80
    S = sum(w * (e * m64).sum(dim=(1, 2, 3)) for (u, e), w in zip(parts, weights)) / msum
    if q < 0:
        return ref, S, L, 2 * sum(w * gamma(5) * float(p.abs().max()) for p, w in zip(preds, weights))
    extra = 0
    for (u, e), p, s, w in zip(parts, preds, scales, weights):
        _, s_lo, s_hi = epe_q_box(u - f64, epe_delta(p, flow, s, zero), eps)
        dev = torch.maximum(s_hi ** q * (1 + POWF_REL) - e, e - s_lo ** q * (1 - POWF_REL))
        extra = extra + w * (dev * m64).sum(dim=(1, 2, 3))
    return ref, S, L, extra / msum * (1 + gamma(L))


def epe_backward_bounds(flow, mask, msum, preds, scales, weights, eps, q, g, zero=None):
    """Per scale (ref, S, pos, L, gpix) of epe_backward_kernel: |got - ref| <= gamma_L S + pos, gpix the signed per-pixel
    gradient w g / msum mask de/du whose transposed Upsample(s) is ref.
    epe_backward_kernel: per lane ceil(cnt / 32) adds of coef * g (coef: 5 roundings, g = d / e: 4), a 5-level shuffle
    tree, * (w g / msum) (3).
    L2 form: the direction d / e of a pixel moves by up to 2 |delta d| / e where delta d, the rounding of the fp32
    up-sampled prediction and difference, is gamma_6 (max |pred| + |flow|).
    q form: g_c = q s^(q-1) sign(d_c); over the box, |g_c| lies in q [s_hi^(q-1), s_lo^(q-1)] widened by powf's error;
    where |d_c| <= delta_c the sign is open (uncertainty q (s^(q-1) + s_lo^(q-1))); where d is exactly 0 (zero) so is g."""
    N, _, H, W = flow.shape
    ps = [p.double().requires_grad_() for p in preds]
    with torch.enable_grad():
        loss, parts = epe_terms(flow, mask, ps, scales, weights, eps, q, zero)
        refs = torch.autograd.grad(loss, ps, g.double())
    kn = (g.double().abs() / msum.double()).view(N, 1, 1, 1)
    ks = (g.double() / msum.double()).view(N, 1, 1, 1)
    m64, f64 = mask.double(), flow.double()
    out = []
    for p, s, w, ref, (u, e) in zip(preds, scales, weights, refs, parts):
        u, e = u.detach(), e.detach()
        Hc, Wc = H // s, W // s
        L = math.ceil((2 * s) ** 2 / 32) + 5 + 9 + 3
        d = u - f64
        if q < 0:
            S = upsample_T(w * kn * m64 * d.abs() / e, s, Hc, Wc)
            M = p.abs().amax(dim=(1, 2, 3), keepdim=True).double()
            pos = upsample_T(w * kn * m64 * 2 * gamma(6) * (M + f64.abs()) / e, s, Hc, Wc)
            gpix = w * ks * m64 * d / e
        else:
            delta = epe_delta(p, flow, s, zero)
            sv, s_lo, s_hi = epe_q_box(d, delta, eps)
            k = q * sv ** (q - 1)
            k_lo, k_hi = q * s_hi ** (q - 1) * (1 - POWF_REL), q * s_lo ** (q - 1) * (1 + POWF_REL)
            unc = torch.where(d.abs() > delta, torch.maximum(k_hi - k, k - k_lo), k + k_hi)
            unc = torch.where((d == 0) & (delta == 0), torch.zeros_like(unc), unc)
            S = upsample_T(w * kn * m64 * k * (d != 0), s, Hc, Wc)
            pos = upsample_T(w * kn * m64 * unc, s, Hc, Wc) * (1 + gamma(L))
            gpix = w * ks * m64 * k * torch.sign(d)
        out.append((ref, S, pos, L, gpix))
    return out


def epe_q_controls(flow, mask, msum, preds, scales, weights, eps, q, g, zero, bounds, loss=None):
    """Near misses of the robust loss, each judged against the bound of the real launch (err / bound, the launch's max):
    the L2 form in place of the q form; the mask rounded to {0, 1} (where that moves at least 1 % of its sum, as after
    the augmentation of a sparse mask); sign(0) = +1 in the q-gradient at the pixels where d is
    exactly 0 (where zero marks some under a nonzero mask).  With loss: the forward's (bounds = epe_forward_bound), else
    the backward's (bounds = epe_backward_bounds)."""
    alts = {"L2 form": (mask, -1.0)}
    if float((mask.round() - mask).abs().sum()) >= 0.01 * float(mask.sum()):
        alts["mask rounded"] = (mask.round(), q)
    res = {}
    for name, (m_alt, q_alt) in alts.items():
        if loss is not None:
            ref, S, L, extra = bounds
            alt = epe_terms(flow, m_alt, [p.double() for p in preds], scales, weights, eps, q_alt, zero)[0]
            res[name] = judge_bound(alt, ref, S, L, extra)[0]
        else:
            alt = epe_backward_bounds(flow, m_alt, msum, preds, scales, weights, eps, q_alt, g, zero)
            res[name] = max(judge_bound(ar[0], r, S, L, pos)[0] for ar, (r, S, pos, L, _) in zip(alt, bounds))
    if loss is None and zero is not None and bool((zero[1] & (mask > 0)).any()):
        s = zero[0]
        i = list(scales).index(s)
        r, S, pos, L, _ = bounds[i]
        N, _, H, W = flow.shape
        ks = (g.double() / msum.double()).view(N, 1, 1, 1)
        plus = weights[i] * ks * mask.double() * q * eps ** (q - 1) * zero[1]
        res["sign(0) = +1"] = judge_bound(r + upsample_T(plus.expand(-1, 2, -1, -1), s, H // s, W // s), r, S, L, pos)[0]
    return res


# ---- image warp (image_warp_bwd.cu): the sampler's slope ---------------------------------------------------------------
def _gather0(img, yi, xi):
    """img[n, c, yi, xi] with 0 outside the plane; yi, xi (N, H, W) integer tensors."""
    N, C, H, W = img.shape
    ok = ((yi >= 0) & (yi < H) & (xi >= 0) & (xi < W)).unsqueeze(1)
    idx = (yi.clamp(0, H - 1) * W + xi.clamp(0, W - 1)).reshape(N, 1, -1).expand(N, C, -1)
    return torch.gather(img.reshape(N, C, -1), 2, idx).view(N, C, *yi.shape[1:]) * ok


def sampler_cell_slopes(img, h, v, y0, x0):
    """d/dh and d/dv (N, C, H, W) of the zero-padded bilinear sample of img at (h, v), taken in the cell with top-left
    corner (y0, x0) (the fractions h - y0, v - x0 may lie a little outside [0, 1]); their S (the same sums on |corners|);
    |Delta| = |a - b - c + d|, the slope of d/dh in the column fraction and of d/dv in the row fraction; sum |corners|."""
    a, b = _gather0(img, y0, x0), _gather0(img, y0, x0 + 1)
    c, d = _gather0(img, y0 + 1, x0), _gather0(img, y0 + 1, x0 + 1)
    ly, lx = (h - y0).unsqueeze(1), (v - x0).unsqueeze(1)
    sy = (1 - lx) * (c - a) + lx * (d - b)
    sx = (1 - ly) * (b - a) + ly * (d - c)
    Sy = (1 - lx).abs() * (a.abs() + c.abs()) + lx.abs() * (b.abs() + d.abs())
    Sx = (1 - ly).abs() * (a.abs() + b.abs()) + ly.abs() * (c.abs() + d.abs())
    return sy, sx, Sy, Sx, (a - b - c + d).abs(), a.abs() + b.abs() + c.abs() + d.abs()


def image_warp_flow_slopes(img, h, v, dh, dv, g, scale, got):
    """err / bound of g_flow_up ((N, 2, H, W), (y, x)) of image_warp_concat_bwd_kernel against float64, and of the
    control that takes every slope from the cell above and to the right.  The kernel's position is the float64 (h, v)
    within (dh, dv); its slope along y is sum_c g_c d sample_c / dh, in the cell of its fp32 position.
    Bound: the dwy / dwx sums (4 fmas), the channel chain (Ci), * scale (1): gamma_(Ci+6) S; the corner weights 1 - l
    and 1 - (1 - l) are off by up to 2u absolutely (2u sum |corners|); and the slope along y is linear in the column
    fraction with slope Delta (continuous across columns), so a column off by dv moves it by |Delta| dv (the larger
    |Delta| of the cells the column may lie in), and the same with the axes swapped.  The slope along y jumps where
    h crosses an integer: where floor(h - dh) != floor(h + dh) the element is accepted against either row cell.
    scale: the factor of both axes, or a (y, x) pair of factors (the stand-alone sampler's grid gradient)."""
    sc = tuple(scale) if isinstance(scale, (tuple, list)) else (scale, scale)
    Ci = img.shape[1]
    L = Ci + 6
    g, ga = g.double(), g.double().abs()
    img = img.double()
    ys = (torch.floor(h - dh).long(), torch.floor(h + dh).long())
    xs = (torch.floor(v - dv).long(), torch.floor(v + dv).long())
    cells = {(i, j): sampler_cell_slopes(img, h, v, ys[i], xs[j]) for i in (0, 1) for j in (0, 1)}
    dmax = torch.stack([c[4] for c in cells.values()]).amax(0)
    cmax = torch.stack([c[5] for c in cells.values()]).amax(0)
    pos_y = abs(sc[0]) * (ga * (dmax * dv.unsqueeze(1) + 2 * U * cmax)).sum(1)
    pos_x = abs(sc[1]) * (ga * (dmax * dh.unsqueeze(1) + 2 * U * cmax)).sum(1)

    # the slope along y in either row cell, each in the column cell of v itself (extrapolating a neighbouring column
    # cell's interpolant across the integer would not be the float64 value); along x the same with the axes swapped
    y0, x0 = torch.floor(h).long(), torch.floor(v).long()
    r, refs = [], []
    for k, pos_k, cand in ((0, pos_y, [sampler_cell_slopes(img, h, v, yy, x0) for yy in ys]),
                           (1, pos_x, [sampler_cell_slopes(img, h, v, y0, xx) for xx in xs])):
        best = None
        for c in cand:
            ref = sc[k] * (g * c[k]).sum(1)
            S = abs(sc[k]) * (ga * c[2 + k]).sum(1)
            rk = _ratio((got[:, k].double() - ref).abs(), gamma(L) * S + pos_k)
            best = rk if best is None else torch.minimum(best, rk)
            refs.append((ref, gamma(L) * S + pos_k))
        r.append(best)
    rr = torch.stack(r)
    i = int(torch.argmax(rr))
    k, e = divmod(i, rr[0].numel())
    pick = lambda t: float(t.reshape(-1)[e])  # noqa: E731
    worst = (f"axis {'yx'[k]} elem {e}: h {pick(h):.9g} v {pick(v):.9g} dh {pick(dh):.3g} dv {pick(dv):.3g} got "
             f"{float(got[:, k].reshape(-1)[e]):.9g} refs " +
             ", ".join(f"{pick(a):.9g} (bound {pick(b):.3g})" for a, b in refs[2 * k:2 * k + 2]))
    nominal = sampler_cell_slopes(img, h, v, y0, x0)
    shifted = sampler_cell_slopes(img, h, v, y0 - 1, x0 + 1)
    ctl = max(float(_ratio(sc[k] * ((g * shifted[k]).sum(1) - (g * nominal[k]).sum(1)).abs(),
                           gamma(L) * abs(sc[k]) * (ga * nominal[2 + k]).sum(1) + pos_k).max())
              for k, pos_k in ((0, pos_y), (1, pos_x)))
    return float(rr.max()), ctl, worst


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
class BackwardRecorder:
    """Wraps the backward of the training graph's autograd Functions, the transposed Upsample and the loss forward; checks
    every launch as it happens."""

    def __init__(self, monkeypatch, run):
        self.run, self.rows, self.failures, self.controls, self.calls = run, [], [], {}, []
        self.capture = None
        self.exact_zero = None      # (scale, bool (N, 1, H, W)): label pixels where the loss kernel's d is exactly 0
        # q form, per scale: (scale, elements with pos > gamma_L S, elements with pos >= S > 0 or pos > S = 0, elements)
        self.epe_vacuous = []
        for cls, fn in ((ops._CorrelationFn, self.correlation), (ops._WarpMaskFn, self.warp_mask),
                        (ops._ImageWarpConcatFn, self.image_warp), (losses._MultiscaleEpeFn, self.epe),
                        (ops._Conv3x3TrainFn, self.conv)):
            orig = cls.backward

            def wrapper(ctx, *grads, _fn=fn, _orig=orig):
                return _fn(_orig, ctx, *grads)
            monkeypatch.setattr(cls, "backward", staticmethod(wrapper))
        self.orig_up, self.orig_call = ops._upsample_backward, ops._call
        self.orig_epe_fwd = losses._MultiscaleEpeFn.forward
        monkeypatch.setattr(ops, "_upsample_backward", self.upsample)
        monkeypatch.setattr(ops, "_call", self._call)
        rec = self

        def epe_forward(ctx, flow, mask, scales, weights, eps, q, *preds):
            return rec.epe_forward(ctx, flow, mask, scales, weights, eps, q, *preds)
        monkeypatch.setattr(losses._MultiscaleEpeFn, "forward", staticmethod(epe_forward))
        orig_warp_fwd = ops._WarpMaskFn.forward

        def warp_forward(ctx, x, flow_c, mask_c, weight, bias, *rest):
            res = orig_warp_fwd(ctx, x, flow_c, mask_c, weight, bias, *rest)
            ctx.test_bias = bias.detach().clone() if bias is not None else None    # not among the saved tensors
            return res
        monkeypatch.setattr(ops._WarpMaskFn, "forward", staticmethod(warp_forward))

    def _call(self, name, dev, *args):
        self.calls.append(name)
        return self.orig_call(name, dev, *args)

    def _row(self, op, name, shape, ratio, err_us, limit=1.0):
        self.rows.append(dict(op=op, name=name, shape=shape, ratio=ratio, err_us=err_us))
        if not ratio <= limit:
            self.failures.append(f"{self.run}: {op} {name} {shape}: err/bound {ratio:.3g}")

    def _control(self, kind, where, ratio):
        self.controls.setdefault(kind, []).append((where, ratio))

    # ---- correlation: corr_bwd_kernel, L = D + 3 ------------------------------------------------------------------
    # acc: one fma per displacement (D roundings), the G tile's LeakyReLU factor g * slope (1), * fl(1/C) (1 + 1 for
    # the rounding of 1/C itself)
    def correlation(self, orig, ctx, go):
        res = orig(ctx, go)
        torch.cuda.synchronize()
        g1, g2 = res[0], res[1]
        d1, d2, out = ctx.saved_tensors
        md, slope = ctx.cfg[2], ctx.cfg[6]
        N, C, H, W = d1.shape
        D = (2 * md + 1) ** 2
        L = D + 3
        worst, worst_us = 0.0, 0.0
        with torch.no_grad():
            for n in range(N):
                gp = go[n:n + 1].double() * torch.where(out[n:n + 1] > 0, 1.0, _f32(slope)).double()
                r1, r2, s1, s2 = corr_bwd_ref(d1[n:n + 1], d2[n:n + 1], gp, md)
                for got, ref, S, side in ((g1, r1, s1, "A"), (g2, r2, s2, "B")):
                    if got is None:
                        continue
                    r, rus, i = judge_bound(got[n:n + 1], ref, S, L)
                    if r > 1.0:
                        self.failures.append(f"{self.run}: corr side {side} n={n} worst at {i}: got "
                                             f"{float(got[n:n + 1].reshape(-1)[i]):.9g} ref {float(ref.reshape(-1)[i]):.9g} "
                                             f"S {float(S.reshape(-1)[i]):.3g}")
                    worst, worst_us = max(worst, r), max(worst_us, rus)
                # one displacement plane dropped (first launch of each md); the LeakyReLU factor dropped, on the first
                # sample with negative outputs (the md=2 correlations of the cascade may have none: there the factor
                # only meets exact zeros at the border, whose gradient is zero)
                ctl = {}
                if n == 0 and f"corr md={md}" not in self.controls:
                    drop = gp.clone()
                    drop[:, D // 2 + 1] = 0
                    ctl[f"corr md={md}"] = drop
                if "corr leaky" not in self.controls and bool((out[n] < 0).any()):
                    ctl["corr leaky"] = go[n:n + 1].double()
                for kind, alt in ctl.items():
                    a1, a2, _, _ = corr_bwd_ref(d1[n:n + 1], d2[n:n + 1], alt, md)
                    self._control(kind, f"md={md} {N}x{C}x{H}x{W}", {kind.split()[-1]: min(
                        judge_bound(a1, r1, s1, L)[0], judge_bound(a2, r2, s2, L)[0])})
        self._row("corr_bwd", f"md={md}", f"{N}x{C}x{H}x{W}", worst, worst_us)
        return res

    # ---- transposed Upsample: upsample_bwd_kernel, L = (2f)^2 + 3 ---------------------------------------------------
    # acc: one add per output pixel read, at most (2f)^2; each term cy * cx * g (cy, cx: one rounding each, 1 - w), * scale
    def upsample(self, go, factor, scale):
        if self.capture is not None:
            self.capture.append(go.detach().clone())
        gi = self.orig_up(go, factor, scale)
        torch.cuda.synchronize()
        N, C, OH, OW = go.shape
        H, W = OH // factor, OW // factor
        L = (2 * factor) ** 2 + 3
        with torch.no_grad():
            ref = upsample_T(go, factor, H, W) * scale
            S = upsample_T(go.abs(), factor, H, W) * abs(scale)
            r, rus, _ = judge_bound(gi, ref, S, L)
            if factor > 1 and f"upsample x{factor}" not in self.controls:
                cut = go.double().clone()
                cut[:, :, factor * (H - 1):] = 0
                cut[:, :, :, factor * (W - 1):] = 0
                self._control(f"upsample x{factor}", f"{N}x{C}x{H}x{W}",
                              {"clamped": judge_bound(upsample_T(cut, factor, H, W) * scale, ref, S, L)[0]})
        self._row("upsample_bwd", f"x{factor}", f"{N}x{C}x{H}x{W}", r, rus)
        return gi

    # ---- fused warp: warp_bwd_pre, deform_bwd_input, deform_bwd_weight, plane_sum -----------------------------------
    def warp_mask(self, orig, ctx, g_out, g_flow_up, g_mask_up):
        self.capture = []
        res = orig(ctx, g_out, g_flow_up, g_mask_up)
        torch.cuda.synchronize()
        captured, self.capture = self.capture, None
        gx, _, _, gw, gb, gtrade = res[:6]
        scale, stride, up, slope, border, has_bias, has_trade = ctx.cfg
        x, weight, out, flow_up, mask_up, conv_out = ctx.saved_tensors
        N, C, H, W = x.shape
        F = weight.shape[0]
        need = ctx.needs_input_grad
        has_mask = mask_up is not None
        total_flow = captured[0] if need[1] else None
        total_mask = captured[1 if need[1] else 0] if (has_mask and need[2]) else None
        det = ops.deterministic()
        name = f"F={F} up={up}" + (" det" if det else "")
        shape = f"{N}x{C}x{H}x{W}"
        P = N * H * W
        L_x0, L_f, L_w, L_b, L_m = F + 8, F + 9 * C + 9, 128 + math.ceil(P / 128) + 10, \
            N * math.ceil(H * W / 256) + 16, F + 5
        worst = {}
        worst_us = {}

        def note(key, r, rus, detail=None):
            worst[key] = max(worst.get(key, 0.0), r)
            worst_us[key] = max(worst_us.get(key, 0.0), rus)
            if r > 1.0 and detail is not None:
                self.failures.append(f"{self.run}: warp {name} {key}: {detail}")

        small = "warp" not in self.controls or P < self.controls["warp"][0][0]
        with torch.no_grad():
            w64 = weight.double()
            sl = _f32(slope)
            gw_ref = torch.zeros_like(w64)
            sgw = torch.zeros_like(w64)
            gb_ref = torch.zeros(F, dtype=torch.float64, device=x.device)
            sgb = torch.zeros_like(gb_ref)
            kappa = 0.0
            ctl_parts = None
            for n in range(N):
                xn, fn = x[n:n + 1], flow_up[n:n + 1]
                gp = g_out[n:n + 1].double() * torch.where(out[n:n + 1] > 0, 1.0, sl)
                if has_trade and gtrade is not None:        # g_tradeoff = fl(g * slope): one rounding
                    note("g_trade", *judge_bound(gtrade[n:n + 1], gp, gp.abs(), 1)[:2])
                if has_mask:
                    sig, es = sigmoid_error(mask_up[n:n + 1].double())
                    kap = float(((es / sig)).max())
                else:
                    sig, es, kap = torch.ones_like(gp[:, :1]), torch.zeros_like(gp[:, :1]), 0.0
                kappa = max(kappa, kap)
                gconv, gabs = gp * sig, gp.abs() * sig
                # conv_out (training forward): deformable convolution + bias before the mask, exact fp32 like the
                # forward's SIMT kernel (test_bench_shapes.py: 2^-20 S)
                if conv_out is not None:
                    cref = 0
                    cS = 0
                    for i, j in TAPS:
                        h, v = _tap_positions(fn, scale, stride, i, j)
                        cref = cref + torch.einsum("fc,nchw->nfhw", w64[:, :, i, j],
                                                   torch_ref.sample_tap(xn.double(), h, v, border))
                        cS = cS + torch.einsum("fc,nchw->nfhw", w64[:, :, i, j].abs(),
                                               torch_ref.sample_tap(xn.double().abs(), h, v, border))
                    b64 = ctx.test_bias.double().view(1, -1, 1, 1) if ctx.test_bias is not None else \
                        torch.zeros((1, F, 1, 1), dtype=torch.float64, device=x.device)
                    r = float(_ratio((conv_out[n:n + 1].double() - cref - b64).abs(), 2.0 ** -20 * (cS + b64.abs())).max())
                    note("conv_out", r, 0.0, f"n={n} conv_out err/bound {r:.3g}")
                    # g_mask: gm = sum_f fma(g_pre, conv) (F), * sig, * (1 - sig) (2), g * slope (1), + g_mask_up (1)
                    if total_mask is not None:
                        cv = conv_out[n:n + 1].double()
                        gm = (gp * cv).sum(1, keepdim=True)
                        gmS = (gp * cv).abs().sum(1, keepdim=True)
                        add = g_mask_up[n:n + 1].double() if (g_mask_up is not None and g_mask_up.numel()) else 0.0
                        ref = gm * sig * (1 - sig) + add
                        S = gmS * sig * (1 - sig) + (add.abs() if torch.is_tensor(add) else 0.0)
                        extra = gmS * (1 - 2 * sig).abs() * es * (1 + gamma(L_m))
                        r, rus, i = judge_bound(total_mask[n:n + 1], ref, S, L_m, extra)
                        note("g_mask", r, rus, f"n={n} elem {i}: got {float(total_mask[n:n + 1].reshape(-1)[i]):.9g} "
                                              f"ref {float(ref.reshape(-1)[i]):.9g}")
                        if small and n == N - 1:
                            last = gp[:, -1:] * cv[:, -1:] * sig * (1 - sig)
                            ctl_parts = {"g_mask": judge_bound(ref - last, ref, S, L_m, extra)[0]}
                gx_r, gf_r, gw_r = warp_bwd_ref(xn, fn, weight, gconv, scale, stride, border)
                sgx, sgf, sgw_n = warp_bwd_S(xn, fn, weight, gabs, scale, stride, border)
                gw_ref += gw_r
                sgw += sgw_n
                gb_ref += gconv.sum(dim=(0, 2, 3))
                sgb += gabs.sum(dim=(0, 2, 3))
                # g_x: gS = F fmas, corner weight (3 roundings), gs * w (1), atomic chain over the n_x contributions the
                # element receives (counted by scattering ones), the sigmoid's error as kappa S
                if gx is not None:
                    n_x = 0
                    for i, j in TAPS:
                        h, v = _tap_positions(fn, scale, stride, i, j)
                        n_x = n_x + corner_scatter(torch.ones_like(h), h, v, H, W)
                    L_x = L_x0 + n_x
                    extra = kap * (1 + gamma(L_x)) * sgx
                    if det:     # det.cuh: n 2^(k+e-62) + u |ref|, B = max_p sum_f |g_conv| * max |W|
                        k_bits = (36 * H * W).bit_length()
                        B = float((gabs.sum(1) * (1 + kap + 2 * F * U)).max()) * float(w64.abs().max())
                        e = math.floor(math.log2(B)) + 1 if B > 0 else -126
                        extra = extra + n_x * 2.0 ** (k_bits + e - 62) + U * gx_r.abs()
                    r, rus, i = judge_bound(gx[n:n + 1], gx_r, sgx, L_x, extra)
                    note("g_x", r, rus, f"n={n} elem {i}: got {float(gx[n:n + 1].reshape(-1)[i]):.9g} ref "
                                        f"{float(gx_r.reshape(-1)[i]):.9g} S {float(sgx.reshape(-1)[i]):.3g}")
                # g_flow (the input of the warp's transposed Upsample): gS (F), the slope (4), the th chain over the
                # channels and the gdy chain over taps and channel blocks (<= 9C), * scale / stride (1), + g_flow_up (1)
                if total_flow is not None:
                    add = g_flow_up[n:n + 1].double() if g_flow_up is not None else 0.0
                    ref = gf_r + add
                    S = sgf + (add.abs() if torch.is_tensor(add) else 0.0)
                    r, rus, i = judge_bound(total_flow[n:n + 1], ref, S, L_f, kap * (1 + gamma(L_f)) * sgf)
                    note("g_flow", r, rus, f"n={n} elem {i}: got {float(total_flow[n:n + 1].reshape(-1)[i]):.9g} "
                                           f"ref {float(ref.reshape(-1)[i]):.9g} S {float(S.reshape(-1)[i]):.3g}")
                if small and n == N - 1:
                    t0 = warp_bwd_ref(xn, fn, weight, gconv, scale, stride, border, taps=((0, 0),))
                    ctl_parts = dict(ctl_parts or {})
                    if gx is not None:
                        ctl_parts["g_x"] = judge_bound(gx_r - t0[0], gx_r, sgx, L_x)[0]
                    if total_flow is not None:
                        ctl_parts["g_flow"] = judge_bound(ref - t0[1], ref, S, L_f)[0]
                    # the last 128-pixel CTA of the launch: the last pixels of this (the last) sample
                    last = torch.zeros_like(gconv)
                    last.view(F, -1)[:, -(P - 128 * ((P - 1) // 128)):] = 1.0
                    last = last * gconv
                    ctl_last_w = warp_bwd_ref(xn, fn, weight, last, scale, stride, border)[2]
                    ctl_last_b = last.sum(dim=(0, 2, 3))
            # g_W: 128-fma chain per CTA, the CTA partials' adds (ceil(P/128)), g_conv (2), the sample (6)
            if gw is not None:
                r, rus, i = judge_bound(gw, gw_ref, sgw, L_w, kappa * (1 + gamma(L_w)) * sgw)
                note("g_W", r, rus, f"elem {i}: got {float(gw.reshape(-1)[i]):.9g} ref {float(gw_ref.reshape(-1)[i]):.9g}")
                if small:
                    ctl_parts["g_W"] = judge_bound(gw_ref - ctl_last_w, gw_ref, sgw, L_w)[0]
            # g_b (plane_sum): per thread N ceil(HW/256) adds, two 5-level shuffle trees, the atomic, g_conv (2)
            if gb is not None:
                r, rus, i = judge_bound(gb, gb_ref, sgb, L_b, kappa * (1 + gamma(L_b)) * sgb)
                note("g_b", r, rus, f"elem {i}: got {float(gb[i]):.9g} ref {float(gb_ref[i]):.9g}")
                if small:
                    ctl_parts["g_b"] = judge_bound(gb_ref - ctl_last_b, gb_ref, sgb, L_b)[0]
        if small and ctl_parts is not None:
            self.controls["warp"] = [(P, f"{name} {shape}", ctl_parts)]
        for key in worst:
            self._row("warp_bwd", f"{name} {key}", shape, worst[key], worst_us[key])
        return res

    # ---- image warp (K5) backward -----------------------------------------------------------------------------------
    def image_warp(self, orig, ctx, g30, g40):
        self.capture = []
        res = orig(ctx, g30, g40)
        torch.cuda.synchronize()
        captured, self.capture = self.capture, None
        gi2 = res[1]
        # the flow's and the mask's inputs of the transposed Upsample(4), in that order
        gfu = captured[0] if res[2] is not None else None
        gmu = captured[-1] if res[3] is not None else None
        i2, fq, mq = ctx.saved_tensors
        scale = ctx.scale
        N, Ci, H, W = i2.shape
        with torch.enable_grad():
            ys = torch.arange(H, dtype=torch.float64, device=i2.device).view(1, H, 1)
            xs = torch.arange(W, dtype=torch.float64, device=i2.device).view(1, 1, W)
            wi = {}
            for n in range(N):
                g = g40[n:n + 1].double()
                disp = torch_ref.upsample(fq[n:n + 1].double(), 4) * scale
                h, v = ys + disp[:, 0], xs + disp[:, 1]
                # the kernel's positions: fl(p + fl(Upsample(4)(flow) * scale)), off by up to 2^-20 (|p| + |d| + 1) px
                # and the fp32 Upsample's own rounding, gamma_8 max |flow| (two interpolations), times the scale
                up_err = gamma(8) * abs(scale) * float(fq[n].abs().max())
                dh, dv = 2.0 ** -20 * (ys + disp[:, 0].abs() + 1), 2.0 ** -20 * (xs + disp[:, 1].abs() + 1)
                dh_f, dv_f = dh + up_err, dv + up_err
                x64 = i2[n:n + 1].double().requires_grad_()
                grid = torch.stack([v / ((W - 1) / 2) - 1, h / ((H - 1) / 2) - 1], dim=-1)
                ref = torch.autograd.grad(tF.grid_sample(x64, grid, align_corners=True), x64, g[:, :Ci])[0]
                S = torch.autograd.grad(tF.grid_sample(x64, grid, align_corners=True), x64, g[:, :Ci].abs())[0]
                # g_im2: atomic chain over the n contributions, the corner weight (3), g * wt (1); each weight is off
                # by up to dh + dv through the position
                gsum = g[:, :Ci].abs()
                cnt = corner_scatter(torch.ones_like(h), h, v, H, W)
                pos = torch.cat([corner_scatter(gsum[:, c] * (dh + dv), h, v, H, W) for c in range(Ci)], 1)
                if gi2 is not None:
                    r, rus, _ = judge_bound(gi2[n:n + 1], ref, S, cnt + 5, pos)
                    wi["g_im2"] = max(wi.get("g_im2", 0.0), r)
                if gfu is not None:
                    with torch.no_grad():
                        r, ctl, worst = image_warp_flow_slopes(i2[n:n + 1], h, v, dh_f, dv_f, g[:, :Ci], scale,
                                                               gfu[n:n + 1])
                    wi["g_flow_up"] = max(wi.get("g_flow_up", 0.0), r)
                    if r > 1.0:
                        self.failures.append(f"{self.run}: image warp g_flow_up n={n}: {worst}")
                    if n == 0 and "image warp" not in self.controls:
                        self._control("image warp", f"{N}x{Ci}x{H}x{W}", {"cell above right": ctl})
                # g_mask_up = g * s (1 - s) (3 roundings); s from an fp32 Upsample(4) (gamma_5 max |mask_q|) and __expf
                m = torch_ref.upsample(mq[n:n + 1].double(), 4)
                s, es = sigmoid_error(m)
                es = es + s * (1 - s) * gamma(5) * float(mq[n].abs().max())
                gm = g[:, Ci:]
                if gmu is not None:
                    r, rus, _ = judge_bound(gmu[n:n + 1], gm * s * (1 - s), (gm * s * (1 - s)).abs(), 3,
                                            gm.abs() * (1 - 2 * s).abs() * es * (1 + gamma(3)))
                    wi["g_mask_up"] = max(wi.get("g_mask_up", 0.0), r)
        for k, r in wi.items():
            self._row("image_warp_bwd", k, f"{N}x{Ci}x{H}x{W}", r, 0.0)
        return res

    # ---- MultiscaleEpe: epe_forward_bound, epe_backward_bounds --------------------------------------------------------
    def epe_forward(self, ctx, flow, mask, scales, weights, eps, q, *preds):
        loss = self.orig_epe_fwd(ctx, flow, mask, scales, weights, eps, q, *preds)
        torch.cuda.synchronize()
        N, _, H, W = flow.shape
        with torch.no_grad():
            bounds = epe_forward_bound(flow, mask, preds, scales, weights, _f32(eps), q, self.exact_zero)
            r, rus, _ = judge_bound(loss, *bounds)
            if q >= 0:
                for kind, ratio in epe_q_controls(flow, mask, None, preds, scales, weights, _f32(eps), q, None,
                                                  self.exact_zero, bounds, loss=loss).items():
                    self._control(f"epe {kind}", f"fwd {N}x{H}x{W}", {"fwd": ratio})
        self._row("epe_fwd", f"{len(preds)} scales" + (f" q={q:g}" if q >= 0 else ""), f"{N}x{H}x{W}", r, rus)
        return loss

    def epe(self, orig, ctx, g):
        res = orig(ctx, g)
        torch.cuda.synchronize()
        flow, mask, msum, *preds = ctx.saved_tensors
        scales, weights, eps, q = ctx.cfg
        grads = res[6:]
        N, _, H, W = flow.shape
        with torch.no_grad():
            bounds = epe_backward_bounds(flow, mask, msum, preds, scales, weights, _f32(eps), q, g, self.exact_zero)
            for s, got, (ref, S, pos, L, gpix) in zip(scales, grads, bounds):
                Hc, Wc = H // s, W // s
                r, rus, _ = judge_bound(got, ref, S, L, pos)
                self._row("epe_bwd", f"x{s}" + (f" q={q:g}" if q >= 0 else ""), f"{N}x2x{Hc}x{Wc}", r, rus)
                if q >= 0:     # elements whose bound the box of the fp32 d dominates / leaves no larger than S
                    self.epe_vacuous.append((s, int((pos > gamma(L) * S).sum()), int(((pos >= S) & (pos > 0)).sum()),
                                             pos.numel()))
                if s == max(scales) and "epe x%d" % s not in self.controls:
                    gd = gpix.clone()
                    gd[:, :, s * (Hc - 1):] = 0
                    gd[:, :, :, s * (Wc - 1):] = 0
                    self._control(f"epe x{s}", f"{N}x2x{Hc}x{Wc}",
                                  {"clamped": judge_bound(upsample_T(gd, s, Hc, Wc), ref, S, L, pos)[0]})
            if q >= 0:
                for kind, ratio in epe_q_controls(flow, mask, msum, preds, scales, weights, _f32(eps), q, g,
                                                  self.exact_zero, bounds).items():
                    self._control(f"epe {kind}", f"bwd {N}x{H}x{W}", {"bwd": ratio})
        return res

    # ---- cuDNN convolution backward: wiring only ----------------------------------------------------------------------
    def conv(self, orig, ctx, g):
        res = orig(ctx, g)
        torch.cuda.synchronize()
        gx, gw, gb = res[:3]
        x, weight, y = ctx.saved_tensors
        slope, dil, stride, has_bias = ctx.cfg
        with torch.no_grad():
            gm = g.double() * torch.where(y > 0, 1.0, _f32(slope)).double()

            def grads(xv, wv, gv, d=dil, s=stride):
                with torch.enable_grad():
                    xr, wr = xv.requires_grad_(), wv.requires_grad_()
                    return torch.autograd.grad(tF.conv2d(xr, wr, stride=s, padding=d, dilation=d), (xr, wr), gv)
            rx, rw = grads(x.double(), weight.double(), gm)
            sx, sw = grads(x.double().abs(), weight.double().abs(), gm.abs())

            def wiring_bound(S):
                # cuDNN's transform-based algorithms (Winograd, FFT) do not keep an exact zero exact: a weight tap that
                # only meets zero data (the outer displacement planes of a 5-row level-6 correlation) comes back as
                # rounding noise of the whole sum, so the bound has a floor at 2^-8 of the tensor's largest S
                return EPS_WIRING * (S + 2.0 ** -8 * S.max())
            worst, zero_err = 0.0, 0.0
            for got, ref, S in ((gx, rx, sx), (gw, rw, sw), (gb, gm.sum(dim=(0, 2, 3)), gm.abs().sum(dim=(0, 2, 3)))):
                if got is not None:
                    err = (got.double() - ref).abs()
                    worst = max(worst, float(_ratio(err, wiring_bound(S)).max()))
                    if bool((S == 0).any()) and float(S.max()) > 0:
                        zero_err = max(zero_err, float(err[S == 0].max() / S.max()))
            if dil > 1 and "conv wiring" not in self.controls and gx is not None:
                cx, _ = grads(x.double(), weight.double(), gm, d=1) if stride == 1 else (None, None)
                if cx is not None:
                    self._control("conv wiring", f"d={dil} {tuple(x.shape)}",
                                  {"dilation 1": float(_ratio((cx - rx).abs(), wiring_bound(sx)).max())})
        # err_us of this row: the largest error where S = 0, relative to the largest S
        self._row("conv_bwd", f"d={dil} s={stride}", "x".join(map(str, x.shape)), worst, zero_err)
        return res

    def report(self):
        for r in self.rows:
            print(f"{self.run:13s} {r['op']:15s} {r['name']:26s} {r['shape']:18s} err/bound={r['ratio']:.3f} "
                  f"err/(uS)={r['err_us']:.3g}")
        for kind, lst in sorted(self.controls.items()):
            for entry in lst:
                where, rs = entry[-2], entry[-1]
                print(f"{self.run:13s} control {kind:14s} on {where}: " +
                      ", ".join(f"{k} err/bound={v:.3g}" for k, v in rs.items()))
        for s, n_dom, n_vac, n in self.epe_vacuous:
            print(f"{self.run:13s} epe_bwd x{s} q form, of {n} elements: pos > gamma_L S at {n_dom} ({n_dom / n:.2e}), "
                  f"pos >= S at {n_vac} ({n_vac / n:.2e})")


RUNS = {   # run: (model class, batch, H, W, image seed, label seed, masked rows from the bottom, deterministic)
    "fwdbwd": (network.MaskFlownetS, 8, 384, 512, 31, 7, 0, False),
    "train8": (network.MaskFlownetS, 4, 576, 960, 32, 8, 36, False),
    "fwdbwd-det": (network.MaskFlownetS, 8, 384, 512, 31, 7, 0, True),
    "cascade-train": (network.MaskFlownet, 2, 384, 512, 33, 9, 0, False),
}


@pytest.mark.gpu
@pytest.mark.parametrize("run", list(RUNS))
def test_every_backward_launch_of_the_benchmarked_step_against_float64(run, monkeypatch):
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
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
