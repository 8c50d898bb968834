"""Per-element error bounds of the census and smoothness losses and their gradients against oracle/unsup_ref.py
(derived in tests/test_unsup_loss.py)."""
import numpy as np
import torch

from oracle import unsup_ref

from .bounds import U

GREY = torch.tensor(unsup_ref.GREY, dtype=torch.float64)
TILE_NT, TILE_PARTS = 256, (8, 32)          # census CTA: 256 pixels of a 32 x 8 tile; smoothness: 256 pixels per CTA
KAPPA_POW, KAPPA_EXP = 4.0, 2.0


def _d64(a):
    return torch.as_tensor(np.asarray(a)).double()


def _grey_and_error(img):
    """I and E_I: 0.2989f etc. (1 rounding each as constants), 3 products, 2 sums, x255 -> 6 roundings of a positive sum."""
    g = unsup_ref.grey(img)
    return g, 6.0 * g.abs()


def census_bounds(img1, img2w, occ, g_loss):
    """float64 (d, coef, loss, g_img2w) of the oracle and their error bounds E (in units of u), from float32 inputs."""
    a, b = _d64(img1), _d64(img2w).requires_grad_(True)
    occ_t = torch.as_tensor(np.asarray(occ))
    N, _, H, W = a.shape
    loss, d, v, coef, vsum = unsup_ref.census_loss(a, b, occ_t)
    if loss.requires_grad:                      # shapes without interior pixels give a constant 0
        (loss * _d64(g_loss)).sum().backward()
    grad = b.grad if b.grad is not None else torch.zeros_like(b)
    d, v, coef, vsum, loss = d.detach(), v.detach(), coef.detach(), vsum.detach(), loss.detach()
    out = {"d": d, "coef": coef, "loss": loss, "vsum": vsum, "grad": grad}
    zero = torch.zeros_like(d)
    if H < 7 or W < 7:
        out.update(E_d=zero, E_coef=zero, E_loss=torch.zeros(N, dtype=torch.float64), E_grad=torch.zeros_like(grad))
        return out
    g1, e1 = _grey_and_error(a.detach())
    g2, e2 = _grey_and_error(b.detach())
    R = unsup_ref.R

    def win(x, dy, dx):      # x(p + o) over the interior
        return x[:, R + dy:H - R + dy, R + dx:W - R + dx]

    def ctr(x):
        return x[:, R:H - R, R:W - R]

    def t_parts(delta, e_delta):
        r = 0.81 + delta * delta
        t = delta / r.sqrt()
        tp = 0.81 / r ** 1.5
        return t, tp * e_delta + 5.0 * t.abs(), tp, -2.43 * delta / r ** 2.5     # d*d, +0.81 (+ its constant), sqrt, /

    E_d = torch.zeros_like(ctr(g1))
    sum_phi = torch.zeros_like(E_d)
    for dy, dx in unsup_ref.OFFSETS:
        D1, D2 = win(g1, dy, dx) - ctr(g1), win(g2, dy, dx) - ctr(g2)
        t1, E_t1, _, _ = t_parts(D1, win(e1, dy, dx) + ctr(e1) + D1.abs())
        t2, E_t2, _, _ = t_parts(D2, win(e2, dy, dx) + ctr(e2) + D2.abs())
        s = t1 - t2
        E_s = E_t1 + E_t2 + s.abs()
        q = 0.1 + s * s
        phi = s * s / q
        E_d = E_d + (0.2 * s / q ** 2).abs() * E_s + 4.0 * phi                        # s*s, +0.1 (+ constant), /
        sum_phi = sum_phi + phi
    E_d = E_d + 47.0 * sum_phi                                                       # 48 terms added in sequence
    pad = lambda x: torch.nn.functional.pad(x, (R, R, R, R))  # noqa: E731
    E_d = pad(E_d)
    dd = d
    qd = dd * dd + unsup_ref.EPS_RHO
    rho = qd ** unsup_ref.P_RHO
    rp = 0.9 * dd * qd ** -0.55
    rpp = 0.9 * qd ** -0.55 - 0.99 * dd * dd * qd ** -1.55
    E_rho = rp.abs() * E_d + (0.45 * 3 + KAPPA_POW) * rho                           # q: d*d, +1e-6f (+ constant); powf
    E_coef = v * (rpp.abs() * E_d + (0.55 * 3 + KAPPA_POW + 2.0) * rp.abs())        # q; powf; 0.9f*d, *pow
    parts = -(-H // TILE_PARTS[0]) * -(-W // TILE_PARTS[1])
    L_sum = TILE_NT + parts + 16                  # a thread's pixels in sequence, the tile's tree, the finishing sums
    E_loss = (v * (E_rho + L_sum * rho)).flatten(1).sum(1) / vsum.clamp(min=1) + loss.abs()
    # backward: G(q) = -sum_o (coef(q+o) + coef(q)) h(q,o), times 255 g / max(vsum, 1), times the channel weight
    cf, ecf = coef, E_coef            # on the whole plane: border pixels receive from their interior neighbours
    gp1 = torch.nn.functional.pad(g1, (R, R, R, R))
    gp2 = torch.nn.functional.pad(g2, (R, R, R, R))
    ep1 = torch.nn.functional.pad(e1, (R, R, R, R))
    ep2 = torch.nn.functional.pad(e2, (R, R, R, R))
    cp, ecp = pad(cf), pad(ecf)
    full = lambda x, dy, dx: x[:, R + dy:R + dy + H, R + dx:R + dx + W]  # noqa: E731
    G_abs = torch.zeros_like(g1)
    E_G = torch.zeros_like(g1)
    for dy, dx in unsup_ref.OFFSETS:
        D1 = full(gp1, dy, dx) - g1
        D2 = full(gp2, dy, dx) - g2
        t1, E_t1, _, _ = t_parts(D1, full(ep1, dy, dx) + e1 + D1.abs())
        E_D2 = full(ep2, dy, dx) + e2 + D2.abs()
        t2, E_t2, tp2, tpp2 = t_parts(D2, E_D2)
        s = t1 - t2
        E_s = E_t1 + E_t2 + s.abs()
        q = 0.1 + s * s
        php = 0.2 * s / q ** 2
        phpp = 0.2 / q ** 2 - 0.8 * s * s / q ** 3
        h = -php * tp2
        E_h = (phpp * tp2).abs() * E_s + (php * tpp2).abs() * E_D2 + 10.0 * h.abs()
        c = full(cp, dy, dx) + cf
        term = c * h
        E_G = E_G + (full(ecp, dy, dx) + ecf) * h.abs() + c.abs() * (E_h + 2.0 * h.abs())
        G_abs = G_abs + term.abs()
    E_G = E_G + 47.0 * G_abs
    k = (255.0 * _d64(g_loss) / vsum.clamp(min=1)).abs().view(N, 1, 1, 1)
    out.update(E_d=E_d, E_coef=E_coef, E_loss=E_loss,
               E_grad=k * GREY.view(1, 3, 1, 1) * (E_G + 6.0 * G_abs).unsqueeze(1))      # 255*(g/max), -acc*, *w (+ const)
    return out


def census_backward_control(img1, img2w, occ, g_loss):
    """The census gradient with the sign of its centre term flipped: sum_o coef(q-o) h(q-o,o) + coef(q) sum_o h(q,o)
    = -sum_o (coef(q+o) - coef(q)) h(q,o), float64."""
    a, b = _d64(img1), _d64(img2w)
    N, _, H, W = a.shape
    _, _, _, coef, vsum = unsup_ref.census_loss(a, b, torch.as_tensor(np.asarray(occ)))
    g1, g2 = unsup_ref.grey(a), unsup_ref.grey(b)
    R = unsup_ref.R
    pd = lambda x: torch.nn.functional.pad(x, (R, R, R, R))  # noqa: E731
    full = lambda x, dy, dx: pd(x)[:, R + dy:R + dy + H, R + dx:R + dx + W]  # noqa: E731
    G = torch.zeros_like(g1)
    for dy, dx in unsup_ref.OFFSETS:
        D2 = full(g2, dy, dx) - g2
        s = unsup_ref.census_t(full(g1, dy, dx) - g1) - unsup_ref.census_t(D2)
        h = -0.2 * s / (0.1 + s * s) ** 2 * 0.81 / (0.81 + D2 * D2) ** 1.5
        G = G - (full(coef, dy, dx) - coef) * h
    k = (255.0 * _d64(g_loss) / vsum.clamp(min=1)).view(N, 1, 1, 1)
    return k * GREY.view(1, 3, 1, 1) * G.unsqueeze(1)


def smoothness_bounds(flow, img, g_loss, kernel_signs=False):
    """float64 (loss, grad) of the oracle and their error bounds E (units of u), from float32 inputs.
    kernel_signs: the gradient takes the sign of each second difference as the kernel evaluates it in fp32,
    fl(fl(lo - 2 mid) + hi) (second_diff in csrc/unsup_loss.cu; 2 mid is exact, so an fma gives the same), instead of
    float64's, and the bound drops its allowance for a sign decided by rounding.  On up-sampled flows most second
    differences are zero in exact arithmetic, and that allowance would cover any error of the size of the gradient."""
    f = _d64(flow).requires_grad_(True)
    f32 = torch.as_tensor(np.asarray(flow)).float()
    im = _d64(img)
    N, _, H, W = f.shape
    loss = unsup_ref.smoothness_loss(f, im)
    if loss.requires_grad:
        (loss * _d64(g_loss)).sum().backward()
    grad = f.grad if f.grad is not None else torch.zeros_like(f)
    f = f.detach()
    parts = -(-H * W // 256)
    L_sum = 256 + parts + 16
    E_S = torch.zeros(N, dtype=torch.float64)
    E_grad = torch.zeros_like(f)
    grad_k = torch.zeros_like(f)
    gl = _d64(g_loss).abs()

    def direction(axis, den):
        nonlocal E_S, E_grad, grad_k
        n_ax = f.shape[axis]
        if n_ax <= 2:
            return
        lo = lambda x: x.narrow(axis, 0, n_ax - 2)  # noqa: E731
        mid = lambda x: x.narrow(axis, 1, n_ax - 2)  # noqa: E731
        hi = lambda x: x.narrow(axis, 2, n_ax - 2)  # noqa: E731
        e = (hi(im) - lo(im)).abs().sum(1)
        arg = -10.0 * (0.5 * (e / 3.0))
        w = torch.exp(arg)
        E_w = w * (5.0 * arg.abs() + KAPPA_EXP)                      # |diff| (1), 2 sums, /3, *10; expf
        D = lo(f) - 2.0 * mid(f) + hi(f)
        E_D = 2.0 * (lo(f).abs() + 2.0 * mid(f).abs() + hi(f).abs())
        term = w * D.abs().sum(1)
        E_term = E_w * D.abs().sum(1) + w * E_D.sum(1) + 2.0 * term
        E_S = E_S + ((E_term + L_sum * term).flatten(1).sum(1) + 4.0 * term.flatten(1).sum(1)) / den
        # backward: each stencil position p contributes tap * w(p) * sign(D(p)) to q in {p-1, p, p+1}
        amb = (D.abs() <= U * E_D).double()                         # the sign may differ from float64's: up to 2 w
        k = gl.view(N, 1, 1, 1) / den
        if kernel_signs:
            amb = torch.zeros_like(amb)
            sgn = torch.sign((lo(f32) - 2 * mid(f32)) + hi(f32)).double()
            ks = _d64(g_loss).view(N, 1, 1, 1) / den
            for shift, tap in ((0, 1.0), (1, -2.0), (2, 1.0)):
                pad = [0, 0, 0, 0]
                pos = 0 if axis == 3 else 2
                pad[pos], pad[pos + 1] = shift, 2 - shift
                grad_k = grad_k + ks * torch.nn.functional.pad(tap * w.unsqueeze(1) * sgn, pad)
        for shift, tap in ((0, 1.0), (1, 2.0), (2, 1.0)):
            contrib = tap * (E_w + 4.0 * w).unsqueeze(1) + tap * 2.0 * w.unsqueeze(1) * amb / U
            pad = [0, 0, 0, 0]
            pos = 0 if axis == 3 else 2
            pad[pos], pad[pos + 1] = shift, 2 - shift
            E_grad = E_grad + k * torch.nn.functional.pad(contrib, pad) + 6.0 * k * torch.nn.functional.pad(
                tap * w.unsqueeze(1).expand_as(D), pad)

    direction(3, 2 * H * (W - 2))
    direction(2, 2 * (H - 2) * W)
    return {"loss": loss.detach(), "grad": grad_k if kernel_signs else grad, "E_loss": E_S + 4.0 * loss.detach().abs(),
            "E_grad": E_grad}


def ratio(got, ref, E):
    """max |got - ref| / (u E / (1 - 64 u)); 0 where both sides agree exactly."""
    got, ref, E = _d64(got), _d64(ref), _d64(E)
    diff = (got - ref).abs()
    bound = U * E / (1 - 64 * U)
    r = torch.where(diff == 0, torch.zeros_like(diff), diff / bound)
    return float(r.max()) if r.numel() else 0.0
