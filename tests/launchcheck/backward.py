"""The float64 checker of the backward launches: error bounds of the correlation, warp, sampler and q-loss gradients.
tests/test_bench_shapes_backward.py derives them."""
import math

import torch

from maskflownet_b200 import ops
from oracle import torch_ref

from .bounds import U, _fp32_positions, _ratio, _warp_offsets

# powf is within 4 ulp over its full range (CUDA C Programming Guide, "Mathematical Functions": single-precision maximum
# ulp errors); one ulp of a normal result is at most 2^-23 of it
POWF_REL = 4 * 2.0 ** -23
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
